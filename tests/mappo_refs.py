"""Float64 restatements of the MAPPO kernels (include/xb200.h, K4M and xb_gae_scan_vn), plus the float32 operation
orders the header claims for the ValueNorm state.  Inputs are numpy arrays; nothing here touches a GPU."""
import numpy as np

F32 = np.float32


def value_norm_update_f32(rm, rmsq, dt, ret, rows_total, beta=0.99999):
    """xb_value_norm_update: ValueNorm.update + running_mean_var in float32, torch's order.  Returns the new
    (rm, rmsq, dt) and (mean, std)."""
    r = np.asarray(ret, np.float64)
    bm, bsq = F32(r.sum() / rows_total), F32((r * r).sum() / rows_total)
    w, omw = F32(beta), F32(1.0 - beta)
    rm = F32(F32(F32(rm) * w) + F32(bm * omw))
    rmsq = F32(F32(F32(rmsq) * w) + F32(bsq * omw))
    dt = F32(F32(F32(dt) * w) + omw)
    return (rm, rmsq, dt), mean_std_f32(rm, rmsq, dt)


def mean_std_f32(rm, rmsq, dt):
    d = max(F32(dt), F32(1e-5))
    mean = F32(F32(rm) / d)
    var = max(F32(F32(F32(rmsq) / d) - F32(mean * mean)), F32(1e-2))
    return mean, F32(np.sqrt(var))


def denorm_f32(x, vn):
    if vn is None:
        return np.asarray(x, np.float32)
    mean, std = vn
    return (np.asarray(x, np.float32) * std + mean).astype(np.float32)


def _denorm_like_torch(x, vn):
    """ValueNorm.denormalize as the reference calls it: a float32 array -> float32; a float64 array (a path whose
    bootstrap was the Python float 0.0, np.append promotes it) -> float64 arithmetic on the float32 (mean, std)."""
    if vn is None:
        return x
    mean, std = vn
    if x.dtype == np.float64:
        return x * np.float64(std) + np.float64(mean)
    return (x * std + mean).astype(np.float32)


def finish_path_ref(rew, val, term, value_next, use_gae, gamma, lam, vn=None):
    """MARL_OnPolicyBuffer.finish_path (memory_tools_marl.py:208-236) for ONE path of one agent, as the reference
    evaluates it: float32 arrays; ``value_next`` an np.float32 (critic output) or the Python float 0.0 (terminal step),
    which np.append turns into a float64 path; Python/numpy float64 scalars.  vn = (mean, std) float32 or None.
    The GAE recursion denormalises scalar by scalar (a 0-d tensor times the [1] float32 state: float32)."""
    rew, val, term = (np.asarray(a, np.float32) for a in (rew, val, term))
    vs = np.append(val, [value_next])
    T = len(rew)
    returns = np.zeros(T, np.float32)
    if use_gae:
        last = 0.0
        dvs = denorm_f32(vs, vn)
        for t in reversed(range(T)):
            d = 1 - int(term[t])
            delta = float(rew[t]) + d * gamma * float(dvs[t + 1]) - float(dvs[t])
            last = delta + d * gamma * lam * last
            returns[t] = last + float(dvs[t])
        adv = returns - _denorm_like_torch(vs[:-1], vn)
    else:
        r_ = np.append(returns, [vs[-1]])
        for t in reversed(range(T)):
            r_[t] = float(rew[t]) + (1 - int(term[t])) * gamma * float(r_[t + 1])
        adv = (r_ - _denorm_like_torch(vs, vn))[:-1]
        returns = r_[:-1]
    return returns.astype(np.float32), adv.astype(np.float32)


def mappo_loss_ref(logits, avail, actions, old_logp, adv, value, old_value, ret, mask, vn, msum, R_total, clip,
                   vclip, hdelta, vf_coef, ent_coef):
    """K4M in float64: (dlogits, dvalue, stats[5] = a_loss, c_loss, entropy, predict_value, loss)."""
    z = np.asarray(logits, np.float64).copy()
    R, A = z.shape
    if avail is not None:
        z[np.asarray(avail)[:, :A] == 0] = -1e10
    m = z.max(1, keepdims=True)
    lse = m + np.log(np.exp(z - m).sum(1, keepdims=True))
    lp = z - lse
    p = np.exp(lp)
    ent = -(p * lp).sum(1)
    a = np.asarray(actions).astype(np.int64)
    logp_a = lp[np.arange(R), a]
    ad = np.asarray(adv, np.float64)
    mk = np.asarray(mask, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        w = mk / msum
        ratio = np.exp(logp_a - np.asarray(old_logp, np.float64))
        lo, hi = 1.0 - clip, 1.0 + clip
        s1, s2 = ratio * ad, np.clip(ratio, lo, hi) * ad
        g1 = np.where(s1 < s2, 1.0, np.where(s1 == s2, 0.5, 0.0))
        g2 = np.where(s2 < s1, 1.0, np.where(s1 == s2, 0.5, 0.0))
        inside = (ratio >= lo) & (ratio <= hi)
        d_logp = -w * ad * (g1 + np.where(inside, g2, 0.0)) * ratio
        onehot = np.zeros_like(z)
        onehot[np.arange(R), a] = 1.0
        dz = d_logp[:, None] * (onehot - p) + (-ent_coef * w)[:, None] * (-p * (lp + ent[:, None]))
        if avail is not None:
            dz[np.asarray(avail)[:, :A] == 0] = 0.0
        vp = np.asarray(value, np.float64)
        r = np.asarray(ret, np.float64)
        tgt = (r - vn[0]) / vn[1] if vn is not None else r

        def L(d):
            if hdelta > 0:
                zz = np.abs(d)
                return (np.where(zz < hdelta, 0.5 * zz * zz, hdelta * (zz - 0.5 * hdelta)),
                        np.clip(d, -hdelta, hdelta))
            return d * d, 2 * d
        l1, gv1 = L(vp - tgt)
        if vclip > 0:
            vo = np.asarray(old_value, np.float64)
            dd = vp - vo
            l2, gv2 = L(vo + np.clip(dd, -vclip, vclip) - tgt)
            lc = np.maximum(l1, l2)
            h1 = np.where(l1 > l2, 1.0, np.where(l1 == l2, 0.5, 0.0))
            h2 = np.where(l2 > l1, 1.0, np.where(l1 == l2, 0.5, 0.0))
            dlc = h1 * gv1 + np.where((dd >= -vclip) & (dd <= vclip), h2 * gv2, 0.0)
        else:
            lc, dlc = l1, gv1
        dv = vf_coef * w * dlc
        a_loss = (-np.minimum(s1, s2) * mk).sum() / msum
        c_loss = (lc * mk).sum() / msum
        e = (ent * mk).sum() / msum
    stats = np.array([a_loss, c_loss, e, vp.sum() / R_total, a_loss + vf_coef * c_loss - ent_coef * e])
    return dz, dv, stats


def mappo_buffer_steps(rng, keys, n_envs, T, obs_dim, A):
    """Seeded inputs of the fixture's buffer cases: T store() dicts in the reference's per-agent layout (env 0 ends a
    path on a terminal step at t = 4), the float32 bootstraps of the final finish_path calls and the targets of the
    ValueNorm update made between the two finish_path rounds."""
    steps = []
    for t in range(T):
        avail = {k: (rng.random((n_envs, A)) > 0.3) for k in keys}
        acts = {}
        for k in keys:
            avail[k][:, 0] = True
            acts[k] = np.array([rng.choice(np.flatnonzero(r)) for r in avail[k]], np.float32)
        steps.append({'obs': {k: rng.normal(size=(n_envs, obs_dim)).astype(np.float32) for k in keys},
                      'actions': acts,
                      'log_pi_old': {k: rng.normal(-1.5, 0.5, n_envs).astype(np.float32) for k in keys},
                      'rewards': {k: rng.normal(0.5, 1.0, n_envs).astype(np.float32) for k in keys},
                      'values': {k: rng.normal(0.0, 2.0, n_envs).astype(np.float32) for k in keys},
                      'terminals': {k: np.array([t == 4, t == 9 and k == keys[1]]) for k in keys},
                      'agent_mask': {k: rng.random(n_envs) > 0.2 for k in keys},
                      'avail_actions': {k: avail[k].astype(np.int64) for k in keys}})
    nexts = [{k: np.float32(rng.normal()) for k in keys} for _ in range(n_envs)]
    return steps, nexts, rng.normal(3.0, 5.0, 30).astype(np.float32)


def mappo_learner_batch(rng, it, B, keys, obs_dim, A):
    """Seeded minibatch of the fixture's learner updates, arrays [n_agents, B, ...] (agent-major, the product's packed
    row order).  Update 1 sets every old log-probability far from any reachable one: all ratios fall outside the clip
    range.  Returns ~ N(3, 20): the normalised targets put Huber(delta = 1) residuals on both sides of delta."""
    n = len(keys)
    avail = rng.random((n, B, A)) > 0.3
    avail[..., 0] = True
    acts = np.array([[rng.choice(np.flatnonzero(r)) for r in avail[i]] for i in range(n)], np.float32)
    old = rng.normal(-1.8, 0.3, (n, B)) if it != 1 else np.where(rng.random((n, B)) < 0.5, -9.0, 3.0)
    return {'obs': rng.normal(size=(n, B, obs_dim)).astype(np.float32), 'actions': acts,
            'log_pi_old': old.astype(np.float32), 'advantages': rng.normal(0, 1, (n, B)).astype(np.float32),
            'values': rng.normal(0, 0.5, (n, B)).astype(np.float32),
            'returns': rng.normal(3, 20, (n, B)).astype(np.float32),
            'agent_mask': rng.random((n, B)) > 0.15, 'avail_actions': avail, 'batch_size': B}

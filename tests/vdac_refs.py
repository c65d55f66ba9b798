"""Float64 restatement of K4V (xb_vdac_loss_fwd_bwd) and the fixture settings shared by tests/golden/make_golden_vdac.py,
tests/oracle_vdac.py and the tests.

* ``k4v_ref``        the kernel's forward and its closed-form gradients in float64 (NumPy): the rules of include/xb200.h K4V;
* ``k4v_autograd``   the reference's expressions (vdac_learner.py:53-122, iac_learner.py:206-252) in float64 torch autograd;
* ``pred_index``     the V_tot index each loss row reads, in the aligned and in the reference's row order.

Rows are in the buffer's (b, i, t) order, r = (b*n + i)*T + t."""
import numpy as np
import torch

FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_T, FIX_B, FIX_HID, FIX_MIX_HID, FIX_HYPER_HID = 3, 8, 5, 6, 6, 4, 16, 8, 16
FIX_UPDATES, FIX_SNAPSHOTS = 4, (1, 3)
# (mixer, use_rnn, use_value_clip, use_huber_loss)
FIX_CASES = [("VDN", True, True, True), ("QMIX", True, True, False), ("IAC", True, False, True),
             ("VDN", False, False, False), ("QMIX", False, True, True), ("IAC", False, True, False)]
SAMPLE_FIELDS = ("obs", "actions", "advantages", "values", "returns", "agent_mask", "avail_actions", "state", "filled")


def case_name(case):
    mixer, use_rnn, clip, huber = case
    return f"{mixer}/rnn{int(use_rnn)}_clip{int(clip)}_huber{int(huber)}"


def case_seed(case):
    return 700 + 10 * FIX_CASES.index(case)


def case_config(case):
    mixer, use_rnn, clip, huber = case
    cfg = dict(agent="IAC" if mixer == "IAC" else "VDAC", use_rnn=use_rnn, use_actions_mask=True,
               use_global_state=False, use_value_clip=clip, value_clip_range=0.2, use_value_norm=False,
               use_huber_loss=huber, huber_delta=1.0, vf_coef=0.5, ent_coef=0.01, gamma=0.99, use_grad_clip=True,
               grad_clip_norm=10.0, learning_rate=7e-4, weight_decay=0, use_linear_lr_decay=False,
               end_factor_lr_decay=0.5, running_steps=96, episode_length=FIX_T, buffer_size=FIX_B, n_epochs=1,
               n_minibatch=1, use_parameter_sharing=True, n_agents=FIX_N, distributed_training=False, use_gae=True,
               gae_lambda=0.95, use_advnorm=False, clip_type=1, parallels=2)
    if mixer != "IAC":
        cfg.update(mixer=mixer, hidden_dim_mixing_net=FIX_MIX_HID, hidden_dim_hyper_net=FIX_HYPER_HID)
    return cfg


def info_keys(mixer):
    g = "shared"
    if mixer == "IAC":
        return ("gradient_norm", f"{g}/actor_loss", f"{g}/critic_loss", f"{g}/entropy", f"{g}/total_loss",
                f"{g}/predict_value", f"{g}/learning_rate")
    return (f"{g}/actor_loss", f"{g}/critic_loss", f"{g}/entropy", f"{g}/predict_value", "gradient_norm",
            "learning_rate", "loss")


def fix_sample(rng, keys, use_rnn, B=FIX_B, T=FIX_T, obs_dim=FIX_OBS, A=FIX_A, S=FIX_S):
    """One batch in the on-policy buffers' sample() layout ({agent: [B, T, ...]} with use_rnn, else [B, ...]): padded
    episodes (filled), agents that die mid-episode (agent_mask 0, only no-op 0 available), random action masks with the
    taken action available, and spread-out values, returns and advantages."""
    shp = (B, T) if use_rnn else (B,)
    L = rng.integers(2, T + 1, size=B)
    L[0] = T
    filled = np.arange(T)[None, :] < L[:, None]
    avail, acts, amask = {}, {}, {}
    for k in keys:
        amask[k] = (np.arange(T)[None, :] < rng.integers(1, 2 * T, size=B)[:, None]) if use_rnn else rng.random(B) > 0.2
        av = rng.random(shp + (A,)) < 0.6
        av[..., 1] = True
        av[~amask[k]] = False
        av[~amask[k], 0] = True
        avail[k] = av.astype(np.float32)
        acts[k] = (rng.random(shp + (A,)) + 10.0 * av).argmax(-1).astype(np.float32)
    f = lambda s: {k: rng.normal(0.0, s, size=shp).astype(np.float32) for k in keys}
    out = {"obs": {k: rng.normal(size=shp + (obs_dim,)).astype(np.float32) for k in keys}, "actions": acts,
           "advantages": f(1.0), "values": f(1.0), "returns": f(2.0), "log_pi_old": f(0.0),
           "rewards": f(1.0), "terminals": {k: np.zeros(shp, bool) for k in keys},
           "agent_mask": amask, "avail_actions": avail,
           "state": rng.normal(size=shp + (S,)).astype(np.float32), "batch_size": B}
    if use_rnn:
        out["filled"], out["sequence_length"] = filled, T
    return out


# ---------------------------------------------------------------- the V_tot a loss row reads
def pred_index(B, n, T, row_order):
    """[R] index into V_tot (b*T + t order) for each row r = (b*n + i)*T + t."""
    r = np.arange(B * n * T)
    if row_order:
        return r // n
    b, t = r // (n * T), r % T
    return b * T + t


def vtot_vdn(value, B, n, T):
    """V_tot(b, t) = sum_i V_i, agents in index order (float64)."""
    return np.asarray(value, np.float64).reshape(B, n, T).sum(1).reshape(-1)


def _huber(d, delta):
    z = np.abs(d)
    return np.where(z < delta, 0.5 * z * z, delta * (z - 0.5 * delta)), np.clip(d, -delta, delta)


def k4v_ref(logits, avail, actions, adv, value, old_value, ret, mask, vn, n, T, mode, row_order, vclip, hdelta,
            vf_coef, ent_coef, M=None, R_total=None):
    """Float64 K4V.  Returns (stats[5] = a_loss, c_loss, e, predict_value, loss; dlogits [R, A]; dvalue)."""
    f = lambda x: None if x is None else np.asarray(x, np.float64)
    logits, adv, ret, mask, old_value = f(logits), f(adv), f(ret), f(mask), f(old_value)
    R, A = logits.shape
    B = R // (n * T)
    M = mask.sum() if M is None else M
    R_total = R if R_total is None else R_total
    z = logits if avail is None else np.where(np.asarray(avail)[:, :A] != 0, logits, -1e10)
    lp = z - z.max(1, keepdims=True)
    lp = lp - np.log(np.exp(lp).sum(1, keepdims=True))
    p = np.exp(lp)
    ent = -(p * lp).sum(1)
    a = np.asarray(actions).astype(np.int64)
    onehot = np.eye(A)[a]
    logp_a = lp[np.arange(R), a]
    with np.errstate(divide="ignore", invalid="ignore"):
        w = mask / M
    dz = (-w * adv)[:, None] * (onehot - p) + (-ent_coef * w)[:, None] * (-p * (lp + ent[:, None]))
    if avail is not None:
        dz = np.where(np.asarray(avail)[:, :A] != 0, dz, 0.0)
    if mode == 0:
        vp = f(value)
    else:
        vt = vtot_vdn(value, B, n, T) if mode == 1 else f(value)
        idx = pred_index(B, n, T, row_order)
        vp = vt[idx]
    tgt = ret if vn is None else (ret - vn[0]) / vn[1]
    sq = lambda d: (d * d, 2 * d)
    L = (lambda d: _huber(d, hdelta)) if hdelta > 0 else sq
    l1, g1 = L(vp - tgt)
    if vclip > 0:
        dd = vp - old_value
        l2, g2 = L(old_value + np.clip(dd, -vclip, vclip) - tgt)
        lc = np.maximum(l1, l2)
        h1 = np.where(l1 > l2, 1.0, np.where(l1 == l2, 0.5, 0.0))
        h2 = np.where(l2 > l1, 1.0, np.where(l1 == l2, 0.5, 0.0))
        dlc = h1 * g1 + np.where((dd >= -vclip) & (dd <= vclip), h2 * g2, 0.0)
    else:
        lc, dlc = l1, g1
    g = vf_coef * w * dlc
    if mode == 0:
        dvalue = g
    else:
        dvt = np.zeros(B * T)
        np.add.at(dvt, idx, g)
        dvalue = dvt if mode == 2 else dvt.reshape(B, 1, T).repeat(n, 1).reshape(-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        a_loss = (-adv * logp_a * mask).sum() / M
        c_loss = (lc * mask).sum() / M
        e = (ent * mask).sum() / M
    stats = np.array([a_loss, c_loss, e, vp.sum() / R_total, a_loss + vf_coef * c_loss - ent_coef * e])
    return stats, dz, dvalue


def reference_loss(lg, avail, actions, adv, v, old_value, ret, mask, n, T, mode, row_order, vclip, hdelta, vf_coef,
                   ent_coef):
    """vdac_learner.py:53-122 / iac_learner.py:206-252 on torch tensors (v: V_i [R], or V_tot [B*T] for mode 2).
    Returns (actor_loss, critic_loss, entropy_loss, pred [R], loss)."""
    R, A = lg.shape
    B = R // (n * T)
    z = lg if avail is None else torch.where(avail[:, :A] != 0, lg, torch.full_like(lg, -1e10))
    dist = torch.distributions.Categorical(logits=z)
    log_pi = dist.log_prob(actions.long())
    actor_loss = -((adv * log_pi) * mask).sum() / mask.sum()
    entropy_loss = (dist.entropy() * mask).sum() / mask.sum()
    if mode == 0:
        pred = v
    else:
        if mode == 1:    # values_tot with VDN_Mixer: agent values of each (b, t) side by side, summed
            vt = v.reshape(B, n, T).transpose(1, 2).reshape(B * T, n).sum(-1, keepdim=True)
        else:
            vt = v.reshape(B * T, 1)
        if row_order:    # AgentGroupedTensor.from_agent_wise({k: values_tot}).packed(group).reshape(-1)
            pred = torch.stack([vt] * n, dim=1).reshape(-1)
        else:
            pred = vt.reshape(B, 1, T).expand(B, n, T).reshape(-1)
    huber = torch.nn.HuberLoss(reduction="none", delta=hdelta) if hdelta > 0 else None
    L = (lambda x: huber(x, ret)) if huber is not None else (lambda x: (x - ret) ** 2)
    if vclip > 0:
        clipped = old_value + (pred - old_value).clamp(-vclip, vclip)
        lc = torch.max(L(pred), L(clipped))
    else:
        lc = L(pred)
    critic_loss = (lc * mask).sum() / mask.sum()
    loss = actor_loss + vf_coef * critic_loss - ent_coef * entropy_loss
    return actor_loss, critic_loss, entropy_loss, pred, loss


def k4v_autograd(logits, avail, actions, adv, value, old_value, ret, mask, n, T, mode, row_order, vclip, hdelta,
                 vf_coef, ent_coef):
    """The reference's expressions in float64 autograd (no ValueNorm).  Returns (stats[5], dlogits, dvalue)."""
    t = lambda x: None if x is None else torch.as_tensor(np.asarray(x, np.float64))
    lg = t(logits).requires_grad_(True)
    v = t(value).requires_grad_(True)
    a, c, e, pred, loss = reference_loss(lg, t(avail), t(actions), t(adv), v, t(old_value), t(ret), t(mask), n, T,
                                         mode, row_order, vclip, hdelta, vf_coef, ent_coef)
    loss.backward()
    stats = np.array([a.item(), c.item(), e.item(), pred.mean().item(), loss.item()])
    return stats, lg.grad.numpy(), v.grad.numpy()

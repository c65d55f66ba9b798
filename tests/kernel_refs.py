"""Float64 restatements of the small fused kernels' contracts as include/xb200.h states them (K3, K4, K6, K7, K8, K9), plus
float32 restatements in the kernels' operation order where the header claims one (DQN td, SAC backup, soft update, the
advantage normalisation given its statistics).  Inputs are NumPy arrays (float32 as the kernels take them); every function
returns NumPy arrays.  tests/test_kernel_refs.py pins these against the oracle's torch formulas on the CPU, and
tests/test_gpu_kernel_edges.py compares the kernels with them."""
import numpy as np

f32, f64 = np.float32, np.float64
EPS32 = 2.0 ** -24          # unit roundoff of float32


def _d(x):
    return np.asarray(x, dtype=f64)


def _log_softmax(z):
    z = _d(z)
    m = z.max(axis=1, keepdims=True)
    return z - (m + np.log(np.exp(z - m).sum(axis=1, keepdims=True)))


def _split(x, y):
    """Gradient share of x in torch.minimum(x, y) / torch.min(x, y): 1 if x < y, 1/2 on a tie, else 0."""
    return np.where(x < y, 1.0, np.where(x == y, 0.5, 0.0))


# ------------------------------------------------------------------------------------------------------ K4
def ppo_loss(logits, value, actions, old_logp, adv, ret, B_total, clip, vf_coef, ent_coef, loss_kind):
    """xb_ppo_loss_fwd_bwd: (dlogits[B,A], dvalue[B], stats[6]) with stats = {a_loss, c_loss, entropy, mean v,
    clip fraction, loss}, every mean a sum over the given rows divided by B_total."""
    lp = _log_softmax(logits)
    p = np.exp(lp)
    B, A = lp.shape
    a = _d(actions).astype(np.int64)
    ent = -(p * lp).sum(axis=1)
    logp_a = lp[np.arange(B), a]
    adv, v, r = _d(adv), _d(value), _d(ret)
    if loss_kind == 0:
        ratio = np.exp(logp_a - _d(old_logp))
        lo, hi = f64(f32(1) - f32(clip)), f64(f32(1) + f32(clip))      # the clip bounds are float32 in the kernel
        s1, s2 = np.clip(ratio, lo, hi) * adv, adv * ratio
        smin = np.minimum(s1, s2)
        inside = (ratio >= lo) & (ratio <= hi)          # clamp backward passes the boundary values
        d_logp = -adv / B_total * (inside * _split(s1, s2) + _split(s2, s1)) * ratio
        clipped = (ratio < lo) | (ratio > hi)
    else:
        smin = adv * logp_a
        d_logp = -adv / B_total
        clipped = np.zeros(B, bool)
    onehot = np.zeros((B, A))
    onehot[np.arange(B), a] = 1.0
    dent = -ent_coef / B_total
    dlogits = d_logp[:, None] * (onehot - p) + dent * (-p * (lp + ent[:, None]))
    dvalue = vf_coef * 2.0 * (v - r) / B_total
    a_loss, c_loss, e = -smin.sum() / B_total, ((v - r) ** 2).sum() / B_total, ent.sum() / B_total
    stats = np.array([a_loss, c_loss, e, v.sum() / B_total, clipped.sum() / B_total,
                      a_loss - ent_coef * e + vf_coef * c_loss])
    return dlogits, dvalue, stats


# ------------------------------------------------------------------------------------------------------ K6
def dqn_target_f32(q_next, q_sel, rew, term, gamma):
    """Float32 target in the kernel's (torch's) order: y = r + (gamma*(1-d))*max, with max = q_next[b, first argmax
    q_sel[b]] for double-Q (q_sel not None)."""
    qn = np.asarray(q_next, f32)
    mx = qn.max(axis=1) if q_sel is None else qn[np.arange(qn.shape[0]), np.argmax(q_sel, axis=1)]
    return np.asarray(rew, f32) + (f32(gamma) * (f32(1) - np.asarray(term, f32))) * mx


def dqn_td(q_eval, q_next, q_sel, actions, rew, term, B_total, gamma):
    """xb_dqn_td_fwd_bwd: (dq[B,A], td_f32[B], td[B], stats[2] = {loss, mean predictQ}); td_f32 is the float32 restatement
    (bit-exact), dq / td / stats are float64 functions of that target."""
    qe = _d(q_eval)
    B = qe.shape[0]
    a = _d(actions).astype(np.int64)
    y32 = dqn_target_f32(q_next, q_sel, rew, term, gamma)
    pred32 = np.asarray(q_eval, f32)[np.arange(B), a]
    td32 = y32 - pred32
    y = _d(rew) + f64(f32(gamma)) * (1.0 - _d(term)) * (_d(q_next).max(axis=1) if q_sel is None else
                                                        _d(q_next)[np.arange(B), np.argmax(q_sel, axis=1)])
    td = y - qe[np.arange(B), a]
    dq = np.zeros_like(qe)
    dq[np.arange(B), a] = -2.0 * td / B_total
    stats = np.array([(td ** 2).sum() / B_total, qe[np.arange(B), a].sum() / B_total])
    return dq, td32, td, stats


# ------------------------------------------------------------------------------------------------------ K8
def sac_actor(log_pi, q1, q2, alpha, B_total):
    """xb_sac_actor_loss: (dlog_pi, dq1, dq2, stats[3] = {Ploss, mean min(q1,q2), mean log_pi})."""
    lp, x, y, a = _d(log_pi), _d(q1), _d(q2), f64(alpha)
    mq = np.minimum(x, y)
    stats = np.array([(a * lp - mq).sum(), mq.sum(), lp.sum()]) / B_total
    return np.full_like(lp, a / B_total), -_split(x, y) / B_total, -_split(y, x) / B_total, stats


def sac_backup_f32(target_q, log_pi_next, rew, term, alpha, gamma):
    """Float32 backup in torch's order: r + ((1-d)*gamma)*(target_q - alpha*log_pi_next)."""
    tv = np.asarray(target_q, f32) - f32(alpha) * np.asarray(log_pi_next, f32)
    return np.asarray(rew, f32) + ((f32(1) - np.asarray(term, f32)) * f32(gamma)) * tv


def sac_critic(q1, q2, target_q, log_pi_next, rew, term, alpha, gamma, B_total):
    """xb_sac_critic_loss: (dq1, dq2, backup, stats[1] = {Qloss}) in float64."""
    y = _d(rew) + (1.0 - _d(term)) * f64(f32(gamma)) * (_d(target_q) - f64(alpha) * _d(log_pi_next))
    e1, e2 = _d(q1) - y, _d(q2) - y
    return 2.0 * e1 / B_total, 2.0 * e2 / B_total, y, np.array([((e1 ** 2).sum() + (e2 ** 2).sum()) / B_total])


# ------------------------------------------------------------------------------------------------------ K9
def qmix_select(q_all, q_tgt, actions, agent_mask, filled, avail, double_q):
    """xb_qmix_select_fwd: (q_eval_taken[B*T,n], q_next_taken[B*T,n], filled_sum).  q_all/q_tgt [B,n,T+1,A], avail
    [B,n,T+1,>=A] (only the first A columns count) or None.  Values are taken from the float32 inputs and multiplied by
    masks in {0, 1}, so the results are exact in float32 as well."""
    B, n, T1, A = q_all.shape
    T = T1 - 1
    NEG = f32(-1e10)
    qe1, qt1 = np.array(q_all[:, :, 1:], f32), np.array(q_tgt[:, :, 1:], f32)
    if avail is not None:
        off = avail[:, :, 1:, :A] == 0
        qe1[off], qt1[off] = NEG, NEG
    if double_q:
        nxt = np.take_along_axis(qt1, np.argmax(qe1, axis=-1)[..., None], -1)[..., 0]
    else:
        nxt = qt1.max(axis=-1)
    a = np.asarray(actions).astype(np.int64)
    taken = np.take_along_axis(np.asarray(q_all[:, :, :T], f32), a[..., None], -1)[..., 0]
    m = np.asarray(agent_mask, f32) * np.asarray(filled, f32)[:, None, :]
    to_rows = lambda x: x.transpose(0, 2, 1).reshape(B * T, n)          # agent-minor [B*T, n]
    return to_rows(taken * m), to_rows(nxt * m), f64(np.asarray(filled, f64).sum())


def qmix_select_bwd(d_taken, actions, agent_mask, filled, A):
    """xb_qmix_select_bwd into a zeroed dq_all[B,n,T+1,A]: only the taken action of steps 0..T-1 is written."""
    B, n, T = np.asarray(actions).shape
    m = np.asarray(agent_mask, f32) * np.asarray(filled, f32)[:, None, :]
    g = np.asarray(d_taken, f32).reshape(B, T, n).transpose(0, 2, 1) * m
    dq = np.zeros((B, n, T + 1, A), f32)
    a = np.asarray(actions).astype(np.int64)
    np.put_along_axis(dq[:, :, :T], a[..., None], g[..., None], -1)
    return dq


def qmix_mix(q, w1, b1, w2, b2, dq_tot, n, H):
    """xb_qmix_mix_fwd/_bwd by float64 autograd of elu(q . |w1| + b1) . |w2| + b2 per row:
    (q_tot[R], dq[R,n], dw1[R,n*H], db1[R,H], dw2[R,H])."""
    import torch
    t = lambda x: torch.tensor(_d(x), dtype=torch.float64, requires_grad=True)
    tq, tw1, tb1, tw2, tb2 = t(q), t(w1), t(b1), t(w2), t(b2)
    R = tq.shape[0]
    hidden = torch.nn.functional.elu(torch.bmm(tq.view(R, 1, n), tw1.view(R, n, H).abs()) + tb1.view(R, 1, H))
    q_tot = (torch.bmm(hidden, tw2.view(R, H, 1).abs()).view(R) + tb2.view(R))
    q_tot.backward(torch.tensor(_d(dq_tot)))
    g = lambda x: x.grad.numpy()
    return q_tot.detach().numpy(), g(tq), g(tw1), g(tb1), g(tw2)


def qmix_td(q_tot, q_tot_next, rewards, terminals, filled, filled_sum, gamma, rows_total):
    """xb_qmix_td: (dq_tot[B*T], stats[2] = {loss_Q, predictQ}).  rewards/terminals [B,n,T]; team reward = mean over
    agents, team terminal = every agent terminal; filled_sum / rows_total are the global sum(filled) and row count."""
    r = _d(rewards).mean(axis=1).reshape(-1)
    d = (np.asarray(terminals) != 0).all(axis=1).reshape(-1).astype(f64)
    f = _d(filled).reshape(-1)
    td = (_d(q_tot) - (r + (1.0 - d) * f64(f32(gamma)) * _d(q_tot_next))) * f
    fs = f64(filled_sum)
    return 2.0 * td * f / fs, np.array([(td ** 2).sum() / fs, _d(q_tot).sum() / rows_total])


# ------------------------------------------------------------------------------------------------------ K7
def grad_norm(g, grad_scale):
    """xb_grad_sumsq: sqrt(sum g^2) * grad_scale."""
    return np.sqrt((_d(g) ** 2).sum()) * f64(f32(grad_scale))


def adam_coef(norm, max_norm, grad_scale):
    """Gradient factor of xb_adam_step, float64: grad_scale * min(1, max_norm / (norm + 1e-6)); max_norm <= 0: no clip."""
    c = f64(f32(grad_scale))
    return c * min(1.0, f64(f32(max_norm)) / (f64(norm) + f64(f32(1e-6)))) if max_norm > 0 else c


def adam_step(p, g, m, v, step_size, bc2_sqrt, beta1, beta2, eps, coef):
    """One float64 Adam step (torch.optim.Adam without weight decay / amsgrad) on g' = g * coef; returns (p, g', m, v)."""
    g = _d(g) * coef
    m = f64(f32(beta1)) * _d(m) + (1.0 - f64(f32(beta1))) * g
    v = f64(f32(beta2)) * _d(v) + (1.0 - f64(f32(beta2))) * g * g
    p = _d(p) - f64(step_size) * m / (np.sqrt(v) / f64(bc2_sqrt) + f64(f32(eps)))
    return p, g, m, v


def soft_update_f32(target, source, tau):
    """xb_soft_update in float32, two roundings per term as torch's tp.mul_(1-tau); tp.add_(tau*ep)."""
    return np.asarray(target, f32) * (f32(1) - f32(tau)) + f32(tau) * np.asarray(source, f32)


# ------------------------------------------------------------------------------------------------------ K3
def adv_stats(x):
    """(mean, population std) of xb_gather_scalars' advantage field, float64."""
    x = _d(x)
    mean = x.mean()
    return mean, np.sqrt(max((x * x).mean() - mean * mean, 0.0))


def adv_normalize_f32(x, stats):
    """xb_adv_normalize in float32 given float32 stats: (x - mean) / (std + 1e-8)."""
    st = np.asarray(stats, f32)
    return (np.asarray(x, f32) - st[0]) / (st[1] + f32(1e-8))

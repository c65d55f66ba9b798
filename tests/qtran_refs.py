"""float64 restatements of the K9Q kernels (QTRAN select, action encoding, three-term loss) and a torch-CPU float64
oracle of one QTRAN_Learner update, written with the reference's own expressions (qtran_learner.py:199-353,
value_factorization.py:354-442, q_mix_head.py:191-292): one-hot, cat, the eye mask of QTRAN_Alt, min / clamp, autograd."""
import numpy as np
import torch
import torch.nn.functional as F

BASE, ALT = 0, 1


def select_ref(q_all, q_tgt, avail, double_q):
    """q_all / q_tgt [B, n, T+1, A] float32, avail [B, n, T+1, A] uint8 or None -> (greedy [B, n, T+1],
    next [B, n, T]) int64: masked first arg-max (value_factorization.py:86-91, qtran_learner.py:262-273)."""
    mq = q_all.clone()
    if avail is not None:
        mq[avail == 0] = -1e10
    greedy = mq.argmax(-1)
    if double_q:
        return greedy, greedy[:, :, 1:]
    mt = q_tgt[:, :, 1:].clone()
    if avail is not None:
        mt[avail[:, :, 1:] == 0] = -1e10
    return greedy, mt.argmax(-1)


def encode_ref(mode, states, t0, h, agent_mask, actions, w1, b1, w2, b2):
    """The Q_jt input of Q_tran (use_rnn): float64, differentiable in h and the weights.  states [B, T+1, S],
    h [B, n, T+1, H], agent_mask [B, n, T], actions [B, n, >= T] (any dtype)."""
    B, n, _, H = h.shape
    T = agent_mask.shape[2]
    D = w1.shape[0]
    A = D - H
    hs = h[:, :, :T] * agent_mask.unsqueeze(-1)
    onehot = F.one_hot(actions[:, :, :T].long(), A).to(h.dtype)
    hs = hs.transpose(1, 2).reshape(-1, n, H)                          # [B*T, n, H]
    onehot = onehot.transpose(1, 2).reshape(-1, n, A)
    u = torch.cat([hs, onehot], dim=-1)
    e = F.linear(torch.relu(F.linear(u, w1, b1)), w2, b2)               # action_encoding
    st = states[:, t0:t0 + T].reshape(B * T, -1)
    if mode == BASE:
        return torch.cat([st, e.sum(dim=1)], dim=-1)
    ids = torch.eye(n, dtype=h.dtype)
    rep = e.unsqueeze(2).repeat(1, 1, n, 1) * (1 - ids).unsqueeze(0).unsqueeze(-1).repeat(e.shape[0], 1, 1, D)
    loo = rep.sum(dim=2)                                                # q_mix_head.py:283-285 (as written)
    x = torch.cat([st.unsqueeze(1).repeat(1, n, 1), loo, ids.unsqueeze(0).repeat(e.shape[0], 1, 1)], dim=-1)
    return x.reshape(B * T * n, -1)


def loss_ref(mode, q_all, actions, greedy, nxt, agent_mask, filled, rewards, terminals, qjt, qjt_g, qjt_n, v, gamma,
             lambda_opt, lambda_nopt):
    """float64 losses of update_rnn (qtran_learner.py:277-343) from the head outputs; differentiable in q_all, qjt and v.
    Layouts as xb_qtran_loss_fwd_bwd.  Returns (loss, stats [5] as a float64 tensor)."""
    B, n, T1, A = q_all.shape
    T = T1 - 1
    m = agent_mask                                                       # [B, n, T]
    q = q_all[:, :, :-1]
    q_a = q.gather(-1, actions.long().unsqueeze(-1)).squeeze(-1) * m     # q_eval_a
    q_g = q.gather(-1, greedy[:, :, :-1].long().unsqueeze(-1)).squeeze(-1) * m
    to_rows = lambda x: x.transpose(1, 2).reshape(B * T, n)             # [B*T, n], row b*T + t
    q_a, q_g = to_rows(q_a), to_rows(q_g)
    r_tot = to_rows(rewards).float().mean(dim=1, keepdim=True).double()
    d_tot = to_rows(terminals).bool().all(1, keepdim=True).double()
    f = filled.reshape(-1, 1).double()
    V = v.reshape(-1, 1)
    q_tot, q_tot_g = q_a.sum(-1, keepdim=True), q_g.sum(-1, keepdim=True)
    if mode == BASE:
        y = r_tot + (1 - d_tot) * gamma * qjt_n.reshape(-1, 1)
        td = (qjt.reshape(-1, 1) - y.detach()) * f
        eo = (q_tot_g - qjt_g.reshape(-1, 1).detach() + V) * f
        en = (q_tot - qjt.reshape(-1, 1).detach() + V).clamp(max=0) * f
        den = f.sum()
        q_joint = qjt.mean()
    else:
        fn = f.repeat(1, n)
        a_rows = to_rows(actions).long().reshape(-1, 1)
        qj = qjt.gather(-1, a_rows).reshape(-1, n)
        qn = qjt_n.gather(-1, to_rows(nxt).long().reshape(-1, 1)).reshape(-1, n)
        qg = qjt_g.gather(-1, to_rows(greedy[:, :, :-1]).long().reshape(-1, 1)).reshape(-1, n)
        y = r_tot + (1 - d_tot) * gamma * qn
        td = (qj - y.detach()) * fn
        eo = (q_tot_g - qg.detach() + V) * fn
        q_count = q.permute(0, 2, 1, 3).reshape(B * T * n, A)
        mask_diag = (1 - torch.eye(n, dtype=q.dtype)).unsqueeze(0).repeat(B * T, 1, 1)
        q_sum_mask = (q_a.unsqueeze(1).repeat(1, n, 1) * mask_diag).sum(-1)
        err = q_count + q_sum_mask.reshape(-1, 1) - qjt.detach() + V.repeat(1, n).reshape(-1, 1)
        en = err.min(dim=-1).values * fn.reshape(-1)
        den = fn.sum()
        q_joint = qj.mean()
    l_td, l_opt, l_nopt = (td ** 2).sum() / den, (eo ** 2).sum() / den, (en ** 2).sum() / den
    loss = l_td + lambda_opt * l_opt + lambda_nopt * l_nopt
    return loss, torch.stack([l_td, l_opt, l_nopt, loss, q_joint]).detach()


def loss_grads(mode, q_all, actions, greedy, nxt, agent_mask, filled, rewards, terminals, qjt, qjt_g, qjt_n, v, gamma,
               lambda_opt, lambda_nopt):
    """(stats, dq_all, dqjt, dv) of loss_ref in float64."""
    q_all, qjt, v = (x.detach().double().requires_grad_(True) for x in (q_all, qjt, v))
    loss, stats = loss_ref(mode, q_all, actions, greedy, nxt, agent_mask.double(), filled, rewards, terminals, qjt,
                           qjt_g.double(), qjt_n.double(), v, gamma, lambda_opt, lambda_nopt)
    loss.backward()
    return stats, q_all.grad, qjt.grad, v.grad


def quantised(rng, shape, scale=64.0):
    """Normal values on a 1/scale grid (exact in float32)."""
    return torch.from_numpy(np.round(rng.normal(size=shape) * scale) / scale).float()

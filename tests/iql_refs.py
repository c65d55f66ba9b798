"""Restatements of K9I (xb_iql_prepare / xb_iql_td_fwd_bwd, include/xb200.h) in the reference's own expressions
(iql_learner.py:37-142 with q_eval sliced outside no_grad and the next-step masks sliced on the time axis, DESIGN.md
section 4; value_factorization.py:86-91 for the masked arg-max).

``forward`` runs in the dtype of its inputs: float64 for the loss and its gradient, float32 for the bit-exact greedy
actions, next values and targets.  ``grads`` is the closed form the kernel writes, checked against autograd of
``forward`` in tests/test_iql.py."""
import numpy as np
import torch


def forward(q_all, q_tgt, actions, rewards, terminals, agent_mask, filled, avail, double_q, gamma):
    """q_all, q_tgt [B,n,T+1,A]; actions, rewards, terminals, agent_mask [B,n,T]; filled [B,T]; avail uint8
    [B,n,T+1,>=A] or None.  Returns (loss, predictQ, next actions [B,n,T], q_next [B*n*T], y [B*n*T], m [B*n*T])."""
    A = q_all.shape[-1]
    q_eval = q_all[:, :, :-1]
    q_eval_next = q_all[:, :, 1:].detach().clone()                     # model_output.actions, steps 1..T
    q_next = q_tgt[:, :, 1:].detach().clone()
    if avail is not None:
        av = avail[:, :, 1:, :A]
        q_eval_next[av == 0] = -1e10
        q_next[av == 0] = -1e10                                         # iql_learner.py:81, time axis sliced
    actions_next = q_eval_next.argmax(dim=-1)
    mask_values = (agent_mask * filled.unsqueeze(1).repeat(1, agent_mask.shape[1], 1)).reshape(-1)
    r, d = rewards.reshape(-1), terminals.reshape(-1)
    q_eval_taken = q_eval.gather(-1, actions.long().unsqueeze(-1)).reshape(-1)
    if double_q:
        q_next_taken = q_next.gather(-1, actions_next.unsqueeze(-1)).reshape(-1)
    else:
        q_next_taken = q_next.max(dim=-1, keepdim=True).values.reshape(-1)
    q_target = r + (1 - d) * gamma * q_next_taken
    td_error = (q_eval_taken - q_target.detach()) * mask_values
    loss = (td_error ** 2).sum() / mask_values.sum()
    return loss, q_eval_taken.mean(), actions_next, q_next_taken, q_target, mask_values


def grads(q_all, q_tgt, actions, rewards, terminals, agent_mask, filled, avail, double_q, gamma):
    """(stats [2] = {loss_Q, predictQ}, dq_all [B,n,T+1,A]) in closed form: 2*td*m/M at the taken action of steps
    0..T-1, zero elsewhere and on step T."""
    loss, pq, _, _, y, m = forward(q_all, q_tgt, actions, rewards, terminals, agent_mask, filled, avail, double_q, gamma)
    B, n, T1, A = q_all.shape
    a = actions.long().reshape(-1)
    q = q_all[:, :, :-1].reshape(-1, A)
    qe = q.gather(-1, a.unsqueeze(-1)).reshape(-1)
    td = (qe - y) * m
    dq = torch.zeros_like(q)
    dq.scatter_(-1, a.unsqueeze(-1), (2 * td * m / m.sum()).unsqueeze(-1))
    out = torch.zeros_like(q_all)
    out[:, :, :-1] = dq.reshape(B, n, T1 - 1, A)
    return torch.stack([loss.detach(), pq.detach()]), out


def inputs(rng, B, n, T, A, masked=True, p_alive=0.8, p_filled=0.85, quantum=None, dtype=np.float32):
    """Random K9I inputs (CPU tensors): q values (on a coarse grid when ``quantum``, so ties are common), available taken
    actions, per-agent rewards and terminals that differ across agents, dead agents and padded steps."""
    def q(shape):
        x = rng.normal(size=shape)
        if quantum:
            x = np.round(x * quantum) / quantum
        return torch.from_numpy(x.astype(dtype))
    q_all, q_tgt = q((B, n, T + 1, A)), q((B, n, T + 1, A))
    avail = None
    if masked:
        av = rng.random((B, n, T + 1, A)) < 0.6
        av[..., rng.integers(0, A)] = True
        avail = torch.from_numpy(av.astype(np.uint8))
        logits = rng.random((B, n, T, A)) + 10.0 * av[:, :, :T]
        actions = logits.argmax(-1)
    else:
        actions = rng.integers(0, A, size=(B, n, T))
    f = lambda x: torch.from_numpy(np.asarray(x, dtype))
    return dict(q_all=q_all, q_tgt=q_tgt, actions=f(actions), rewards=f(rng.normal(size=(B, n, T))),
                terminals=f(rng.random((B, n, T)) < 0.15), agent_mask=f(rng.random((B, n, T)) < p_alive),
                filled=f(rng.random((B, T)) < p_filled), avail=avail)

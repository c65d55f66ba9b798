"""Float64 restatements of the K9W Weighted QMIX kernels (xb_wqmix_select_fwd / _bwd, xb_wqmix_loss_fwd_bwd) and the
fixture shared by tests/golden/make_golden_wqmix.py, the oracle test and the GPU tests.  Pure torch on the CPU.

select_ref / select_bwd_ref / loss_ref state what include/xb200.h (K9W) specifies, in float64; the CPU tests check the
loss gradients against torch autograd and the GPU tests check the kernels against these functions."""
import numpy as np
import torch

NEG = -1e10
OW, CW = 0, 1


def masked_argmax(q, avail):
    """First maximal index over the last axis with unavailable actions at -1e10 (avail None: all available).  Runs on
    float32 values as the kernel compares them (the -1e10 replacement is a float32 constant there)."""
    q = q.to(torch.float32)
    if avail is not None:
        q = torch.where(avail != 0, q, torch.tensor(NEG, dtype=torch.float32))
    # torch.argmax returns the first maximal index
    return q.argmax(dim=-1)


def select_ref(q_all, q_cent, q_cent_tgt, q_tgt, actions, agent_mask, filled, avail, double_q):
    """q_* [B,n,T+1,A]; actions, agent_mask [B,n,T]; filled [B,T]; avail [B,n,T+1,A] or None.  Returns float64
    q_eval_taken, q_cent_taken, q_next_cent [B*T, n], greedy int64 [B,n,T], agree bool [B*T], filled_sum (float64)."""
    B, n, T1, A = q_all.shape
    T = T1 - 1
    g_all = masked_argmax(q_all, avail)                                   # [B, n, T+1]
    g = g_all[:, :, :-1]
    nxt = g_all[:, :, 1:] if double_q else q_tgt[:, :, 1:].to(torch.float32).argmax(dim=-1)
    a = actions.long()
    m = agent_mask.double() * filled.double().unsqueeze(1)               # [B, n, T]
    take = lambda q, idx: q.double().gather(-1, idx.unsqueeze(-1)).squeeze(-1)
    q_eval = take(q_all[:, :, :-1], a) * m
    q_c = take(q_cent[:, :, :-1], g) * m
    q_n = take(q_cent_tgt[:, :, 1:], nxt) * m
    rows = lambda x: x.permute(0, 2, 1).reshape(B * T, n)               # agent-minor
    agree = ((g == a) & (m != 0)).all(dim=1).reshape(B * T)
    return rows(q_eval), rows(q_c), rows(q_n), g, agree, filled.double().sum()


def select_bwd_ref(d_eval, d_cent, actions, greedy, agent_mask, filled, A):
    """Scatter of the two differentiable selections: dq_all, dq_cent [B,n,T+1,A] float64."""
    B, n, T = actions.shape
    m = agent_mask.double() * filled.double().unsqueeze(1)
    cols = lambda d: d.double().reshape(B, T, n).permute(0, 2, 1) * m   # [B, n, T]
    out = []
    for d, idx in ((d_eval, actions.long()), (d_cent, greedy.long())):
        z = torch.zeros(B, n, T + 1, A, dtype=torch.float64)
        z[:, :, :-1].scatter_(-1, idx.unsqueeze(-1), cols(d).unsqueeze(-1))
        out.append(z)
    return out


def team_targets(rewards, terminals, q_ff_next, gamma):
    """y = mean_i r + (1 - all_i d) * gamma * q_ff_next per row (float64)."""
    B, n, T = rewards.shape
    r = rewards.double().mean(dim=1).reshape(B * T)
    d = (terminals != 0).all(dim=1).double().reshape(B * T)
    return r + (1.0 - d) * gamma * q_ff_next.double()


def weights(mode, alpha, td, y, q_ff, agree):
    one = (td < 0) if mode == OW else (agree.bool() | (y > q_ff))
    return torch.where(one, torch.ones_like(td), torch.full_like(td, alpha))


def loss_ref(q_tot, q_ff, q_ff_next, rewards, terminals, filled, agree, filled_sum, mode, alpha, gamma, rows_total):
    """Closed form of K9W loss: (dq_tot, dq_ff, stats[4]) in float64; filled_sum / rows_total are the global ones."""
    f = filled.double().reshape(-1)
    y = team_targets(rewards, terminals, q_ff_next, gamma)
    qt, qf = q_tot.double(), q_ff.double()
    td, dc = qt - y, qf - y
    w = weights(mode, alpha, td, y, qf, agree)
    fs = float(filled_sum)
    lq, lc = (w * td * td * f).sum() / fs, (dc * dc * f).sum() / fs
    stats = torch.stack([lq, lc, lq + lc, qt.sum() / rows_total])
    return 2.0 * w * td * f / fs, 2.0 * dc * f / fs, stats


def loss_autograd(q_tot, q_ff, q_ff_next, rewards, terminals, filled, agree, mode, alpha, gamma):
    """The reference's loss expressions (wqmix_learner.py:166-199) under torch autograd, float64, one shard."""
    qt = q_tot.double().clone().requires_grad_(True)
    qf = q_ff.double().clone().requires_grad_(True)
    f = filled.double().reshape(-1)
    y = team_targets(rewards, terminals, q_ff_next, gamma)
    td = qt - y.detach()
    w = weights(mode, alpha, td.detach(), y, qf.detach(), agree)
    loss_central = (((qf - y.detach()) ** 2) * f).sum() / f.sum()
    loss_qmix = (w.detach() * (td ** 2) * f).sum() / f.sum()
    loss = loss_qmix + loss_central
    loss.backward()
    stats = torch.stack([loss_qmix.detach(), loss_central.detach(), loss.detach(), qt.detach().mean()])
    return qt.grad, qf.grad, stats


# ---------------------------------------------------------------- the reference-update fixture (wqmix_update.npz)
FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_T, FIX_B = 3, 12, 7, 10, 8, 6
FIX_HID = 16                       # fc_hidden_sizes, recurrent_hidden_size, q_hidden_size
FIX_MIX, FIX_HYPER, FIX_FF = 8, 8, 16
FIX_UPDATES = 4
FIX_SNAPSHOTS = (1, 3)             # updates after which the fixture holds the whole state_dict (sync_frequency = 2)
FIX_CASES = [(agent, dq) for agent in ("OWQMIX", "CWQMIX") for dq in (True, False)]
FIX_INFO_KEYS = ("loss_Qmix", "loss_central", "loss", "predictQ", "learning_rate")


def fix_case_seed(agent, double_q):
    return 100 + 10 * (agent == "CWQMIX") + int(double_q)


def fix_learner_config(agent, double_q):
    """Learner keys shared by the reference run and the product (as a dict: the callers add device and the rest)."""
    return dict(agent=agent, episode_length=FIX_T, use_grad_clip=False, grad_clip_norm=0.5, parallels=4,
                running_steps=100000, start_training=0, n_epochs=1, use_parameter_sharing=True, use_rnn=True,
                use_actions_mask=True, learning_rate=7e-4, sync_frequency=2, double_q=double_q, gamma=0.99, alpha=0.1,
                end_factor_lr_decay=0.5, use_linear_lr_decay=True, distributed_training=False)


def fix_sample(rng, keys=None, B=FIX_B, T=FIX_T, obs_dim=FIX_OBS, A=FIX_A, S=FIX_S):
    """One padded episode batch in the replay's sample() layout: episodes of random length (padded steps have
    filled = 0), agents that die mid-episode (agent_mask = 0 from then on, only action 0 available), random action masks
    with action 1 always available to the living, and taken actions that are available."""
    keys = keys or [f"agent_{i}" for i in range(FIX_N)]
    L = rng.integers(max(2, T // 2), T + 1, size=B)
    L[0] = T
    filled = np.arange(T)[None, :] < L[:, None]
    death = {k: rng.integers(1, 2 * T, size=B) for k in keys}           # step at which the agent dies (often never)
    avail, acts, amask = {}, {}, {}
    for k in keys:
        av = rng.random((B, T + 1, A)) < 0.6
        av[..., 1] = True
        amask[k] = np.arange(T)[None, :] < death[k][:, None]
        av[~np.concatenate([amask[k], amask[k][:, -1:]], axis=1)] = False  # a dead agent can only take no-op 0
        av[~np.concatenate([amask[k], amask[k][:, -1:]], axis=1), 0] = True
        avail[k] = av.astype(np.float32)
        logits = rng.random((B, T, A)) + 10.0 * av[:, :T]
        acts[k] = logits.argmax(-1).astype(np.float32)
    return {"obs": {k: rng.normal(size=(B, T + 1, obs_dim)).astype(np.float32) for k in keys},
            "actions": acts,
            "rewards": {k: rng.normal(size=(B, T)).astype(np.float32) for k in keys},
            "terminals": {k: (rng.random((B, T)) < 0.1) for k in keys},
            "agent_mask": amask, "avail_actions": avail, "filled": filled,
            "state": rng.normal(size=(B, T + 1, S)).astype(np.float32), "batch_size": B, "sequence_length": T}

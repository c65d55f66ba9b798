"""Float64 restatements of the K6Z kernels (xb_dist_greedy / xb_c51_loss_fwd_bwd / xb_qrdqn_loss_fwd_bwd), the
reference's float32 torch expressions whose results the kernels reproduce bit for bit (C51's Tz and projection weights,
QR's backup), and the seeded inputs of the C51 / QR-DQN tests and fixture."""
import numpy as np
import torch


# ------------------------------------------------------------------------------------------------- float64 references
def _softmax(x):
    m = x.max(axis=-1, keepdims=True)
    e = np.exp(x - m)
    return e / e.sum(axis=-1, keepdims=True)


def greedy_ref(z, supports=None):
    """-> (first argmax [B], Q [B, A], C51 probabilities [B, A, N] or None), in float64."""
    z = np.asarray(z, np.float64)
    if supports is None:
        q = z.mean(axis=-1)
        return q.argmax(axis=-1), q, None
    p = _softmax(z)
    q = (p * np.asarray(supports, np.float64)).sum(-1)
    return q.argmax(axis=-1), q, p


def c51_ref(z_eval, z_next, supports, actions, rew, ter, gamma, v_min, v_max, B_total):
    """c51_learner.py:38-51 in float64 -> (dlogits [B, A, N], target action [B], loss share, Tz [B, N], target [B, N])."""
    z = np.asarray(supports, np.float64)
    N = z.shape[0]
    dz = (v_max - v_min) / (N - 1)
    ta, _, pn = greedy_ref(z_next, supports)
    B = len(ta)
    pt = pn[np.arange(B), ta]
    rew, ter = np.asarray(rew, np.float64), np.asarray(ter, np.float64)
    tz = np.clip(rew[:, None] + gamma * z[None, :] * (1.0 - ter[:, None]), v_min, v_max)
    proj = np.clip(1.0 - np.abs(tz[:, :, None] - z[None, None, :]) / dz, 0.0, 1.0)
    target = np.einsum("bj,bji->bi", pt, proj)
    a = np.asarray(actions).astype(np.int64)
    p = _softmax(np.asarray(z_eval, np.float64)[np.arange(B), a])
    loss = -(target * np.log(p + 1e-8)).sum(-1).sum() / B_total
    g = -target / (p + 1e-8) / B_total
    d = np.zeros(np.shape(z_eval))
    d[np.arange(B), a] = p * (g - (p * g).sum(-1, keepdims=True))
    return d, ta, loss, tz, target


def qrdqn_ref(z_eval, z_next, actions, rew, ter, gamma, B_total):
    """qrdqn_learner.py:40-48 in float64 -> (dq [B, A, N], target action [B], loss share, backup [B, N])."""
    ta, _, _ = greedy_ref(z_next)
    zn = np.asarray(z_next, np.float64)
    B, A, N = zn.shape
    th = zn[np.arange(B), ta]
    y = np.asarray(rew, np.float64)[:, None] + gamma * th * (1.0 - np.asarray(ter, np.float64)[:, None])
    a = np.asarray(actions).astype(np.int64)
    x = np.asarray(z_eval, np.float64)[np.arange(B), a]
    d = np.zeros((B, A, N))
    d[np.arange(B), a] = 2.0 * (x - y) / (B_total * N)
    return d, ta, ((x - y) ** 2).sum() / (B_total * N), y


# --------------------------------------------------------------------------------- the reference's float32 expressions
def torch_tz(rew, ter, supports, gamma, v_min, v_max):
    """c51_learner.py:46-47."""
    nxt = rew.unsqueeze(1) + gamma * supports * (1 - ter.unsqueeze(1))
    return nxt.clamp(v_min, v_max)


def torch_projection(tz, supports, delta_z):
    """c51_learner.py:49-50: the [B, N(j), N(i)] weights clamp(1 - |Tz_j - z_i| / delta_z, 0, 1)."""
    return (1 - (tz.unsqueeze(-1) - supports.unsqueeze(0)).abs() / delta_z).clamp(0, 1)


def torch_qr_backup(rew, ter, theta, gamma):
    """qrdqn_learner.py:46."""
    return rew.unsqueeze(1) + gamma * theta * (1 - ter.unsqueeze(1))


def torch_c51_loss(z_eval, z_next, supports, actions, rew, ter, gamma, v_min, v_max, delta_z):
    """c51_learner.py:38-51 over raw logits with autograd (the reference's expressions); returns (loss, target action)."""
    N = supports.shape[0]
    tz = torch.softmax(z_next, -1)
    ta = (supports * tz).sum(-1).argmax(-1)
    pe = torch.softmax(z_eval, -1)
    cur = pe.gather(1, actions.long().reshape(-1, 1, 1).expand(-1, -1, N)).squeeze(1)
    tgt = tz.gather(1, ta.reshape(-1, 1, 1).expand(-1, -1, N)).squeeze(1).detach()
    proj = torch_projection(torch_tz(rew, ter, supports, gamma, v_min, v_max), supports, delta_z)
    tgt = torch.bmm(tgt.unsqueeze(1), proj).squeeze(1)
    return -(tgt * torch.log(cur + 1e-8)).sum(1).mean(), ta


def torch_qrdqn_loss(z_eval, z_next, actions, rew, ter, gamma):
    """qrdqn_learner.py:40-48 with autograd."""
    N = z_eval.shape[-1]
    ta = z_next.mean(-1).argmax(-1)
    cur = z_eval.gather(1, actions.long().reshape(-1, 1, 1).expand(-1, -1, N)).squeeze(1)
    tgt = z_next.gather(1, ta.reshape(-1, 1, 1).expand(-1, -1, N)).squeeze(1)
    tgt = torch_qr_backup(rew, ter, tgt, gamma)
    return torch.nn.functional.mse_loss(tgt.detach(), cur), ta


# ------------------------------------------------------------------------------------------------------------ inputs
def supports_of(v_min, v_max, N):
    """C51DeepQNetwork.supports as the model builds it (torch.linspace on the CPU, float32)."""
    return torch.linspace(v_min, v_max, N)


def loss_batch(rng, B, A, N, v_min=-10.0, v_max=10.0):
    """Raw head outputs with duplicated action rows (ties), atoms whose softmax underflows to 0, rewards large enough that
    Tz clamps at both ends, rows with ter = 1, and one reward placing Tz exactly on an atom."""
    ze = rng.normal(0.0, 2.0, (B, A, N)).astype(np.float32)
    zn = rng.normal(0.0, 2.0, (B, A, N)).astype(np.float32)
    if A > 1:
        zn[::5, 1] = zn[::5, 0]                      # ties: the first index wins
    ze[1::7, :, 0] = -1000.0                         # exp underflows, in float32 and in float64: p = 0 exactly
    zn[2::7, :, N - 1] = -1000.0
    rew = rng.normal(0.0, 0.6 * (v_max - v_min), B).astype(np.float32)
    ter = (rng.random(B) < 0.25).astype(np.float32)
    ter[0] = 1.0
    rew[0] = np.float32(v_min + (v_max - v_min) / (N - 1))       # ter = 1: Tz is this atom, exactly
    act = rng.integers(0, A, B).astype(np.float32)
    return dict(z_eval=ze, z_next=zn, actions=act, rew=rew, ter=ter)


# ---------------------------------------------------------------------------------------------------------- fixture
OBS, HIDDEN, N_ACT, B_FIX = 6, 32, 3, 40
ATOMS, QUANTILES, V_MIN, V_MAX = 51, 20, -10, 10
GAMMA, LR, SYNC, N_UPDATES, CLIP_NORM = 0.97, 1e-3, 2, 4, 0.05


def fixture_batch(rng):
    """One update batch: 6-d observations, rewards large enough that Tz clamps at both v_min and v_max, 25 % terminal
    rows and one terminal row for certain."""
    term = (rng.random(B_FIX) < 0.25).astype(np.float32)
    term[0] = 1.0
    rew = rng.normal(0.0, 6.0, B_FIX).astype(np.float32)
    rew[1], rew[2] = 25.0, -25.0
    return {"obs": rng.normal(0.0, 1.0, (B_FIX, OBS)).astype(np.float32),
            "actions": rng.integers(0, N_ACT, B_FIX).astype(np.float32),
            "obs_next": rng.normal(0.0, 1.0, (B_FIX, OBS)).astype(np.float32), "rewards": rew, "terminals": term}


def fixture_state_dict(sd, seed=47):
    """``helpers.seeded_state_dict`` values with every target network a copy of its live network (the reference's
    deepcopy) and C51's ``supports`` left as built."""
    from helpers import seeded_state_dict
    out = seeded_state_dict(sd, seed)
    for k in list(out):
        if k == "supports":
            out[k] = sd[k].clone()
        for t in ("target_representation.", "target_Z_head."):
            if k.startswith(t):
                src = {"target_representation.": "representation.", "target_Z_head.": "eval_Z_head."}[t]
                out[k] = out[src + k[len(t):]].clone()
    return out

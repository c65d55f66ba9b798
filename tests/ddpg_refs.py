"""Float64 restatements of the K8T kernels (xb_perturb_actions / xb_ddpg_critic_loss / xb_ddpg_actor_loss), the torch
expressions of the reference whose float32 results the kernels reproduce bit for bit, and the seeded inputs of the DDPG /
TD3 tests and fixture."""
import numpy as np
import torch


# ------------------------------------------------------------------------------------------------- float64 references
def perturb_ref(a, noise, scale, noise_clip, low, high):
    n = np.asarray(noise, np.float64) * scale
    if noise_clip >= 0:
        n = np.clip(n, -noise_clip, noise_clip)
    return np.clip(np.asarray(a, np.float64) + n, np.asarray(low, np.float64), np.asarray(high, np.float64))


def critic_ref(q1, q2, tq1, tq2, rew, term, gamma, B_total):
    """-> dq1, dq2 (None for DDPG), backup, stats (Qloss, mean q1, mean q2): the local rows' shares over B_total rows."""
    f = lambda x: None if x is None else np.asarray(x, np.float64)
    q1, q2, tq1, tq2, rew, term = map(f, (q1, q2, tq1, tq2, rew, term))
    t = tq1 if tq2 is None else np.minimum(tq1, tq2)
    y = rew + gamma * (1.0 - term) * t
    e1 = q1 - y
    st = [(e1 ** 2).sum() / B_total, q1.sum() / B_total, 0.0]
    dq2 = None
    if q2 is not None:
        e2 = q2 - y
        dq2 = 2.0 * e2 / B_total
        st[0] += (e2 ** 2).sum() / B_total
        st[2] = q2.sum() / B_total
    return 2.0 * e1 / B_total, dq2, y, np.array(st)


def actor_ref(q1, q2, B_total):
    """-> dq1, dq2 (None for DDPG), Ploss share."""
    q1 = np.asarray(q1, np.float64)
    if q2 is None:
        return np.full_like(q1, -1.0 / B_total), None, -q1.sum() / B_total
    q2 = np.asarray(q2, np.float64)
    d = np.full_like(q1, -0.5 / B_total)
    return d, d.copy(), -((q1 + q2) / 2.0).sum() / B_total


# --------------------------------------------------------------------------------- the reference's float32 expressions
def torch_exploration(a, noise, scale, low, high):
    """core/off_policy.py:143-144 with the noise supplied."""
    return torch.clamp(a + noise * scale, low, high)


def torch_smoothing(a, noise, sigma, clip, low, high):
    """actor_critic.py:292-295 with the noise supplied."""
    n = (noise * sigma).clamp(-clip, clip)
    return torch.maximum(torch.minimum(a + n, high), low)


def torch_backup(rew, term, gamma, tq1, tq2=None):
    """td3_learner.py:51 (ddpg_learner.py:48 multiplies in the other order: the same float32 product)."""
    t = tq1 if tq2 is None else torch.minimum(tq1, tq2)
    return rew + gamma * (1 - term) * t


# ------------------------------------------------------------------------------------------------------------ inputs
def loss_batch(rng, B, nan_rows=0):
    f = lambda: rng.normal(0.0, 1.0, B).astype(np.float32)
    d = dict(q1=f(), q2=f(), tq1=f(), tq2=f(), rew=f(), term=(rng.random(B) < 0.25).astype(np.float32))
    d["q2"][1::3] = d["q1"][1::3]
    d["tq2"][::4] = d["tq1"][::4]
    d["term"][:1] = 1.0
    if nan_rows:
        d["tq1"][:nan_rows] = np.nan
    return d


def action_batch(rng, B, D, low, high):
    """Actions inside and outside [low, high], and noise with large entries (some |sigma*n| exceed any clip)."""
    a = rng.uniform(-1.5, 1.5, (B, D)).astype(np.float32) * np.maximum(np.abs(low), np.abs(high)).astype(np.float32)
    return a.astype(np.float32), (rng.normal(0.0, 1.0, (B, D)) * 1.5).astype(np.float32)


def bounds(D):
    low = -np.linspace(0.5, 2.0, D).astype(np.float32)
    high = np.linspace(0.25, 2.0, D).astype(np.float32)
    return low, high


# ---------------------------------------------------------------------------------------------------------- fixture
OBS, ACT, HIDDEN, B_FIX = 8, 3, 32, 48
LOW = np.array([-1.0, -0.5, -2.0], np.float32)     # the tanh output alone crosses the bounds of the middle component
HIGH = np.array([1.0, 0.25, 2.0], np.float32)
SIGMA, NOISE_CLIP = 0.6, 0.5                       # |SIGMA*n| > NOISE_CLIP for |n| > 0.83
DELAY, N_UPDATES, CLIP_NORM = 2, 4, 0.05


def fixture_batch(rng):
    """One update batch of the fixture: 8-d observations (scaled up in the first half so the tanh saturates), actions
    inside the bounds, normal rewards, 25 % terminal rows and one terminal row for certain."""
    def obs():
        o = rng.normal(0.0, 1.0, (B_FIX, OBS))
        o[:B_FIX // 2] *= 8.0
        return o.astype(np.float32)
    term = (rng.random(B_FIX) < 0.25).astype(np.float32)
    term[0] = 1.0
    return {"obs": obs(), "actions": rng.uniform(LOW, HIGH, (B_FIX, ACT)).astype(np.float32), "obs_next": obs(),
            "rewards": rng.normal(0.0, 1.0, B_FIX).astype(np.float32), "terminals": term}


def fixture_state_dict(sd, seed=43):
    """``helpers.seeded_state_dict`` values with every target network a copy of its live network (the reference's
    deepcopy)."""
    from helpers import seeded_state_dict
    out = seeded_state_dict(sd, seed)
    for k in list(out):
        for t in ("target_actor.", "target_critic."):
            if k.startswith(t):
                out[k] = out[t[len("target_"):] + k[len(t):]].clone()
    return out


def fixture_noise(seed):
    """The standard normal draw of TD3's Qtarget at the update whose generator was seeded with ``seed``."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B_FIX, ACT, generator=g).numpy()

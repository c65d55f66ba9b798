"""Float64 restatements of the K8D kernels (xb_sacdis_actor_loss / xb_sacdis_critic_loss) and the seeded inputs of the
SAC-Discrete tests and fixture.

The policy probabilities are those of the reference, Categorical(logits).probs = softmax(logits - logsumexp(logits)),
computed by torch in ``prob_dtype`` (float32 for the kernels: which entries underflow to 0 or to a subnormal is a float32
fact); everything after them is float64.  log_pi = log(p + 1e-8*[p == 0]) (actor_critic.py:184-205)."""
import numpy as np
import torch


def probs_of(logits, prob_dtype=torch.float32):
    z = torch.as_tensor(np.asarray(logits)).to(prob_dtype)
    return torch.distributions.Categorical(logits=z).probs.double().numpy()


def log_rule(p):
    return np.log(p + 1e-8 * (p == 0.0))


def sacdis_actor_ref(logits, q1, q2, alpha, B_total, prob_dtype=torch.float32):
    """-> dlogits [B, A], stats (Ploss, Qvalue, mean log_pi): the local rows' shares of the means over B_total rows."""
    p = probs_of(logits, prob_dtype)
    lp = log_rule(p)
    mq = np.minimum(np.asarray(q1, np.float64), np.asarray(q2, np.float64))
    t = alpha * lp - mq
    g = t + alpha * p / (p + 1e-8 * (p == 0.0))
    dz = p * (g - (p * g).sum(1, keepdims=True)) / B_total
    A = p.shape[1]
    stats = np.array([(p * t).sum() / B_total, mq.sum() / (B_total * A), lp.sum() / (B_total * A)])
    return dz, stats


def sacdis_critic_ref(q1, q2, actions, logits_next, tq1, tq2, rew, term, alpha, gamma, B_total,
                      prob_dtype=torch.float32):
    """-> dq1, dq2 (dense [B, A]), backup [B], Qloss share.  A row whose action is not in [0, A) selects no column: zero
    gradient rows and a NaN loss."""
    p = probs_of(logits_next, prob_dtype)
    tq = np.minimum(np.asarray(tq1, np.float64), np.asarray(tq2, np.float64))
    target = (p * (tq - alpha * log_rule(p))).sum(1)
    backup = np.asarray(rew, np.float64) + (1.0 - np.asarray(term, np.float64)) * gamma * target
    B, A = p.shape
    a = np.trunc(np.asarray(actions, np.float64))
    ok = (a >= 0) & (a < A)
    rows = np.arange(B)
    ai = np.where(ok, a, 0).astype(np.int64)
    e1 = np.where(ok, np.asarray(q1, np.float64)[rows, ai] - backup, np.nan)
    e2 = np.where(ok, np.asarray(q2, np.float64)[rows, ai] - backup, np.nan)
    dq1, dq2 = np.zeros((B, A)), np.zeros((B, A))
    dq1[rows[ok], ai[ok]] = 2.0 * e1[ok] / B_total
    dq2[rows[ok], ai[ok]] = 2.0 * e2[ok] / B_total
    return dq1, dq2, backup, float(((e1 ** 2).sum() + (e2 ** 2).sum()) / B_total)


def edge_logits(rng, B, A, scale=2.0):
    """Random logits whose leading rows reach the float32 edges of the probability rule: an entry 120 below the row's
    max (p underflows to exactly 0), one 95 below (a subnormal p), both at once, and for A = 1 the single-action row."""
    z = rng.normal(0.0, scale, (B, A))
    if A >= 2:
        for r, gaps in enumerate(((120.0,), (95.0,), (120.0, 95.0), (200.0, 150.0))):
            if r >= B:
                break
            for j, gap in enumerate(gaps[:A - 1]):
                z[r, (j + 1) % A] = z[r].max() - gap
    return z.astype(np.float32)


def edge_batch(rng, B, A):
    """Inputs of both kernels with the edge rows above, rows with q1 == q2 and terminal rows."""
    f = lambda *s: rng.normal(0.0, 1.0, s).astype(np.float32)
    logits, logits_next = edge_logits(rng, B, A), edge_logits(rng, B, A)
    q1, q2, tq1, tq2 = f(B, A), f(B, A), f(B, A), f(B, A)
    q2[1::3] = q1[1::3]                   # ties of min(q1, q2)
    tq2[::4] = tq1[::4]
    actions = rng.integers(0, A, B).astype(np.float32)
    rew = f(B)
    term = (rng.random(B) < 0.25).astype(np.float32)
    term[:2] = 1.0
    return dict(logits=logits, q1=q1, q2=q2, actions=actions, logits_next=logits_next, tq1=tq1, tq2=tq2, rew=rew,
                term=term)


# ---------------------------------------------------------------------------------------------------------- fixture
OBS, A_FIX, HIDDEN, B_FIX = 8, 5, 32, 48
OBS_SCALES = (1.0, 1.0, 30.0, 60.0, 120.0, 400.0)   # some observation rows scaled up: their logits spread far apart


def fixture_batch(rng):
    """One SACDIS_Learner.update batch of the fixture: 8-d observations (a sixth of the rows at each scale of
    OBS_SCALES), A = 5 actions stored as float32, normal rewards and 25 % terminal rows."""
    def obs():
        o = rng.normal(0.0, 1.0, (B_FIX, OBS))
        o *= np.repeat(np.array(OBS_SCALES), B_FIX // len(OBS_SCALES))[:, None]
        return o.astype(np.float32)
    return {"obs": obs(), "actions": rng.integers(0, A_FIX, B_FIX).astype(np.float32), "obs_next": obs(),
            "rewards": rng.normal(0.0, 1.0, B_FIX).astype(np.float32),
            "terminals": (rng.random(B_FIX) < 0.25).astype(np.float32)}


def fixture_state_dict(sd, seed=41):
    """The fixture's initial weights: ``helpers.seeded_state_dict`` values, with the second critic tower a copy of the
    first except for every other output bias of its head (so that q1 == q2 in those columns at the first update), and
    the target critic a copy of the critic, as the reference's deepcopy leaves it."""
    from helpers import seeded_state_dict
    out = seeded_state_dict(sd, seed)
    for k in list(out):
        if k.startswith("critic.representation_2."):
            out[k] = out[k.replace("representation_2", "representation_1")].clone()
        elif k.startswith("critic.critic_head_2."):
            out[k] = out[k.replace("critic_head_2", "critic_head_1")].clone()
    last_bias = sorted(k for k in out if k.startswith("critic.critic_head_2.") and k.endswith(".bias"))[-1]
    out[last_bias][::2] += 0.25
    for k in list(out):
        if k.startswith("target_critic."):
            out[k] = out["critic." + k[len("target_critic."):]].clone()
    return out

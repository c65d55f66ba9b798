"""Float64 restatements of the Gaussian-policy kernels' contracts as include/xb200.h states them - K4G
(xb_ppo_gauss_loss_fwd_bwd) and K10G (xb_gaussian_act) - in the manner of tests/kernel_refs.py, whose helpers they reuse, and
the seeded inputs of the Gaussian PPO fixture (tests/golden/ppo_gauss_update.npz).  Inputs are NumPy arrays (float32 as the
kernels take them); every function returns NumPy arrays.  tests/test_gauss_ppo.py pins the references against torch
autograd and DiagGaussianDistribution on the CPU, and tests/test_gpu_gauss_ppo.py compares the kernels with them."""
import numpy as np

from kernel_refs import EPS32, _d, _split, f32, f64  # noqa: F401  (EPS32 re-exported for the GPU tolerances)


# ------------------------------------------------------------------------------------------------------ K4G
LOG_SQRT_2PI = 0.5 * np.log(2.0 * np.pi)


def gauss_logp_terms(mu, log_std, x):
    """Per-component float64 log N(x; mu, exp(log_std)) [B,D] and z = (x - mu) / sigma."""
    ls = _d(log_std)[None, :]
    z = (_d(x) - _d(mu)) / np.exp(ls)
    return -0.5 * z * z - ls - LOG_SQRT_2PI, z


def ppo_gauss_loss(mu, log_std, value, actions, old_logp, adv, ret, B_total, clip, vf_coef, ent_coef, loss_kind):
    """xb_ppo_gauss_loss_fwd_bwd: (dmu[B,D], dlog_std[D], dvalue[B], stats[6]); stats as ppo_loss, the ratio / clamp /
    minimum rules as K4, Normal(mu, exp(log_std)) log-prob and entropy summed over the D components."""
    terms, z = gauss_logp_terms(mu, log_std, actions)
    logp = terms.sum(axis=1)
    B, D = terms.shape
    ent = np.full(B, (0.5 + LOG_SQRT_2PI + _d(log_std)).sum())
    adv, v, r = _d(adv), _d(value), _d(ret)
    if loss_kind == 0:
        ratio = np.exp(logp - _d(old_logp))
        lo, hi = f64(f32(1) - f32(clip)), f64(f32(1) + f32(clip))
        s1, s2 = np.clip(ratio, lo, hi) * adv, adv * ratio
        smin = np.minimum(s1, s2)
        inside = (ratio >= lo) & (ratio <= hi)
        d_logp = -adv / B_total * (inside * _split(s1, s2) + _split(s2, s1)) * ratio
        clipped = (ratio < lo) | (ratio > hi)
    else:
        smin = adv * logp
        d_logp = -adv / B_total
        clipped = np.zeros(B, bool)
    sig = np.exp(_d(log_std))[None, :]
    dmu = d_logp[:, None] * z / sig
    dlog_std = (d_logp[:, None] * (z * z - 1.0)).sum(axis=0) - ent_coef * B / B_total
    dvalue = vf_coef * 2.0 * (v - r) / B_total
    a_loss, c_loss, e = -smin.sum() / B_total, ((v - r) ** 2).sum() / B_total, ent.sum() / B_total
    stats = np.array([a_loss, c_loss, e, v.sum() / B_total, clipped.sum() / B_total,
                      a_loss - ent_coef * e + vf_coef * c_loss])
    return dmu, dlog_std, dvalue, stats


# ------------------------------------------------------------------------------------------------------ K10G
def gaussian_act(mu, log_std, noise=None, forced=None):
    """xb_gaussian_act in float64: (actions[N,D] or None in forced mode, logp[N], entropy[N])."""
    sig = np.exp(_d(log_std))[None, :]
    if forced is not None:
        x, out = _d(forced), None
    else:
        x = _d(mu) + sig * _d(noise) if noise is not None else _d(mu).copy()
        out = x
    terms, _ = gauss_logp_terms(mu, log_std, x)
    N = terms.shape[0]
    return out, terms.sum(axis=1), np.full(N, (0.5 + LOG_SQRT_2PI + _d(log_std)).sum())


# ------------------------------------------------------------------------------------------------------ fixture inputs
def ppo_gauss_samples(rng, it, B, obs_dim, act_dim):
    """The inputs of update ``it`` of tests/golden/make_golden_gauss.py and of the tests that replay it: a Box
    minibatch for a Gaussian policy with log_std near 0.  old_logp sits near the log-density of such actions; update 1
    shifts it by +-2 so that most of its ratios leave the clip range on both sides."""
    obs = rng.normal(size=(B, obs_dim)).astype(np.float32)
    acts = np.clip(rng.normal(size=(B, act_dim)) * 0.5, -1, 1).astype(np.float32)
    old = (rng.normal(size=B) * 0.1 - act_dim * (0.125 + 0.5 * np.log(2 * np.pi))).astype(np.float32)
    if it == 1:
        old = (old + np.where(rng.random(B) < 0.5, -2.0, 2.0)).astype(np.float32)
    return {"obs": obs, "actions": acts, "returns": rng.normal(size=B).astype(np.float32),
            "advantages": rng.normal(size=B).astype(np.float32), "aux_batch": {"old_logp": old}}

"""Float64 restatements of K4N (xb_npg_loss_fwd_bwd, xb_npg_gauss_loss_fwd_bwd) and K7N (xb_npg_natural_grad) as
include/xb200.h states them, the reference's own expressions (npg_learner.py:37-43, 100-113) in torch for the autograd
and dense-inverse comparisons, and the constants of the reference fixture tests/golden/npg_update.npz.  NumPy, no GPU."""
import numpy as np
import torch
from torch.distributions import Categorical, Normal

LAM = 1e-3                      # npg_learner.py:111


def _stats(adv, logp, v, ret):
    adv, logp, v, ret = (np.asarray(x, np.float64) for x in (adv, logp, v, ret))
    B = len(v)
    return np.array([-(adv * logp).sum() / B, ((v - ret) ** 2).sum() / B, v.sum() / B, logp.sum(), 0, 0, 0, 0])


def cat_ref(z, v, act, adv, ret):
    """-> (dlogits, dscore [B, A], dvalue [B], stats[8], sum log pi)."""
    z = np.asarray(z, np.float64)
    B, A = z.shape
    m = z.max(-1, keepdims=True)
    lp = z - (m + np.log(np.exp(z - m).sum(-1, keepdims=True)))
    a = np.asarray(act).astype(np.int64)
    onehot = np.eye(A)[a]
    dscore = onehot - np.exp(lp)
    adv = np.asarray(adv, np.float64)
    dlogits = -(adv / B)[:, None] * dscore
    logp = lp[np.arange(B), a]
    dvalue = 2.0 * (np.asarray(v, np.float64) - np.asarray(ret, np.float64)) / B
    return dlogits, dscore, dvalue, _stats(adv, logp, v, ret), logp.sum()


def gauss_ref(mu, log_std, v, x, adv, ret):
    """-> (dmu, dlog_std [D], smu [B, D], slog_std [D], dvalue, stats[8], sum log pi)."""
    mu, ls, x = (np.asarray(t, np.float64) for t in (mu, log_std, x))
    B = mu.shape[0]
    sig = np.exp(ls)
    z = (x - mu) / sig
    logp = (-0.5 * z * z - ls - 0.5 * np.log(2 * np.pi)).sum(-1)
    smu, sls_rows = z / sig, z * z - 1.0
    adv = np.asarray(adv, np.float64)
    c = -(adv / B)[:, None]
    dvalue = 2.0 * (np.asarray(v, np.float64) - np.asarray(ret, np.float64)) / B
    return (c * smu, (c * sls_rows).sum(0), smu, sls_rows.sum(0), dvalue, _stats(adv, logp, v, ret), logp.sum())


def torch_npg_terms(out, v, act, adv, ret, gaussian):
    """npg_learner.py:38-43 on raw outputs: ``out`` = logits, or (mu, log_std).  -> (sum log pi, a_loss, c_loss)."""
    if gaussian:
        mu, ls = out
        logp = Normal(mu, ls.exp(), validate_args=False).log_prob(act).sum(-1)
    else:
        logp = Categorical(logits=out, validate_args=False).log_prob(act.long())
    a_loss = -(adv * logp).mean()
    c_loss = torch.nn.functional.mse_loss(v, ret)
    return logp.sum(), a_loss, c_loss


def natural_grad_ref(g, s, kappa, lam=LAM):
    """K7N's closed form in float64: (g - s kappa (s.g) / (lam + kappa s.s)) / lam."""
    g, s = np.asarray(g, np.float64).ravel(), np.asarray(s, np.float64).ravel()
    return (g - s * (kappa * (s @ g) / (lam + kappa * (s @ s)))) / lam


def dense_ref(g, s, kappa, lam=LAM):
    """The reference's F^-1 g with F = outer(s, s) kappa + lam I, inverted densely in float64."""
    g, s = torch.as_tensor(np.asarray(g, np.float64).ravel()), torch.as_tensor(np.asarray(s, np.float64).ravel())
    F = torch.outer(s, s) * kappa + lam * torch.eye(len(s), dtype=torch.float64)
    return (torch.linalg.inv(F) @ g).numpy()


def conditioning(s, kappa, lam=LAM):
    """(lam + kappa s.s) / lam: the eigenvalue ratio of F along s, whose magnitude bounds F's condition number."""
    s = np.asarray(s, np.float64).ravel()
    return (lam + kappa * (s @ s)) / lam


# ------------------------------------------------------------------------------------------------ reference fixture
FIX_OBS, FIX_HIDDEN, FIX_ROWS, FIX_A, FIX_D, FIX_UPDATES = 4, 12, 24, 3, 2, 4
FIX_LR, FIX_CLIP_NORM = 1e-2, 0.5
FIX_CASES = [(kind, mb, clip) for kind in ("cat", "gauss") for mb in (1, 2) for clip in (0, 1)]
FIX_INFO_KEYS = ["actor-loss", "critic-loss", "learning_rate_actor", "learning_rate_critic", "predict_value"]


def fix_learner_config(mb, clip):
    """The learner keys of a fixture case: horizon_size = the rows (so kappa's divisor differs from B when mb = 2) and
    running_steps = the update count, so the LinearLR schedules reach their end inside the case."""
    return dict(learning_rate=FIX_LR, use_grad_clip=bool(clip), grad_clip_norm=FIX_CLIP_NORM, end_factor_lr_decay=0.5,
                horizon_size=FIX_ROWS, parallels=1, running_steps=FIX_UPDATES, n_epochs=1, n_minibatch=mb)


def fix_rows(kind, seed):
    rng = np.random.default_rng(seed)
    obs = rng.normal(size=(FIX_ROWS, FIX_OBS)).astype(np.float32)
    # Box actions at the initial policy's scale (exp(log_std) = exp(-1)), as acting draws them: far-off actions make
    # |lam + kappa s.s| / lam, and with it the error of the reference's float32 inverse, several orders larger
    act = ((rng.normal(size=(FIX_ROWS, FIX_D)) * np.exp(-1.0)).astype(np.float32) if kind == "gauss"
           else rng.integers(0, FIX_A, FIX_ROWS).astype(np.float32))
    adv = rng.normal(size=FIX_ROWS).astype(np.float32)
    ret = rng.normal(size=FIX_ROWS).astype(np.float32)
    return obs, act, adv, ret


def fix_indices(mb, seed):
    """The minibatches of the FIX_UPDATES updates: each epoch a fresh permutation cut into ``mb`` parts."""
    rng = np.random.default_rng(seed + 1)
    out = []
    while len(out) < FIX_UPDATES:
        perm = rng.permutation(FIX_ROWS)
        out += list(perm.reshape(mb, -1))
    return np.stack(out[:FIX_UPDATES])


def fix_case_seed(kind, mb, clip):
    return 500 + 10 * (kind == "gauss") + 2 * mb + clip

"""Float64 restatements of the two K4P losses (xb_ppg_aux_loss_fwd_bwd, xb_ppg_aux_gauss_loss_fwd_bwd) and their
gradients, term by term as include/xb200.h states them, plus the reference's own expressions (ppg_learner.py:127-131)
in torch for the autograd comparison.  NumPy, no GPU."""
import numpy as np
import torch
import torch.nn.functional as F
from torch.distributions import Categorical, Normal, kl_divergence


def _lse(x):
    """torch.logsumexp(dim=-1, keepdim=True): an infinite max is replaced by 0 before the shift."""
    m = x.max(-1, keepdims=True)
    m = np.where(np.isinf(m), 0.0, m)
    return np.log(np.exp(x - m).sum(-1, keepdims=True)) + m


def _softmax(x):
    m = x.max(-1, keepdims=True)
    e = np.exp(x - m)
    return e / e.sum(-1, keepdims=True)


def _value_terms(v, aux, ret, B_total):
    v, ret = np.asarray(v, np.float64), np.asarray(ret, np.float64)
    dvalue = 2.0 * (v - ret) / B_total
    if aux is None:
        return dvalue, None, 0.0, ((v - ret) ** 2).sum() / B_total
    aux = np.asarray(aux, np.float64)
    return dvalue, -2.0 * (v - aux) / B_total, ((v - aux) ** 2).sum() / B_total, ((v - ret) ** 2).sum() / B_total


def _stats(aux_loss, kl_loss, value_loss, v, kl_beta, B_total):
    return np.array([aux_loss, kl_loss, value_loss, aux_loss + kl_beta * kl_loss + value_loss,
                     np.asarray(v, np.float64).sum() / B_total, 0, 0, 0])


def cat_aux_ref(z, o, v, aux, ret, kl_beta, B_total=None):
    """-> (dlogits [B, A] or None, dvalue, daux or None, stats[8], kl per row or None).  ``z is None``: the critic-only
    form (value_loss alone)."""
    B = len(v)
    B_total = B if B_total is None else B_total
    dvalue, daux, aux_loss, value_loss = _value_terms(v, aux, ret, B_total)
    if z is None:
        return None, dvalue, daux, _stats(aux_loss, 0.0, value_loss, v, kl_beta, B_total), None
    with np.errstate(all="ignore"):
        z, o = np.asarray(z, np.float64), np.asarray(o, np.float64)
        lse_p = _lse(z)
        lp, lq = z - lse_p, o - _lse(o)
        p, q = _softmax(lp), _softmax(lq)
        d = lp - lq
        t = np.where(p == 0, 0.0, np.where(q == 0, np.inf, p * d))
        kl = t.sum(-1)
        c = kl_beta / B_total
        g = np.where((p == 0) | (q == 0), 0.0, c)
        dp = g * d                                            # 0 * inf = NaN, as autograd
        s1 = (p * dp).sum(-1, keepdims=True)
        G = p * (dp - s1) + g * p
        dz = G - np.exp(z - lse_p) * G.sum(-1, keepdims=True)
    kl_loss = kl.sum() / B_total
    return dz, dvalue, daux, _stats(aux_loss, kl_loss, value_loss, v, kl_beta, B_total), kl


def gauss_aux_ref(mu, log_std, old_mu, old_log_std, v, aux, ret, kl_beta, B_total=None):
    """-> (dmu [B, D], dlog_std [D], dvalue, daux, stats[8], kl [B, D])."""
    B, D = np.shape(mu)
    B_total = B if B_total is None else B_total
    dvalue, daux, aux_loss, value_loss = _value_terms(v, aux, ret, B_total)
    with np.errstate(all="ignore"):
        mu, omu = np.asarray(mu, np.float64), np.asarray(old_mu, np.float64)
        s, so = np.exp(np.asarray(log_std, np.float64)), np.exp(np.asarray(old_log_std, np.float64))
        r = s / so
        vr = r * r
        x = (mu - omu) / so
        kl = 0.5 * (vr + x * x - 1.0 - np.log(vr))
        h = 0.5 * kl_beta / (B_total * D)
        dmu = h * 2.0 * x / so
        dls = B * ((h - h / vr) * 2.0 * r / so * s)
    kl_loss = kl.sum() / (B_total * D)
    return dmu, dls, dvalue, daux, _stats(aux_loss, kl_loss, value_loss, v, kl_beta, B_total), kl


def torch_cat_aux_loss(z, o, v, aux, ret, kl_beta):
    """ppg_learner.py:127-131 for Categorical(logits=) on both sides: (loss, aux_loss, kl_loss, value_loss)."""
    p = Categorical(logits=z, validate_args=False)
    q = Categorical(logits=o, validate_args=False)
    aux_loss = F.mse_loss(v.detach(), aux)
    kl_loss = kl_divergence(p, q).mean()
    value_loss = F.mse_loss(v, ret)
    return aux_loss + kl_beta * kl_loss + value_loss, aux_loss, kl_loss, value_loss


def torch_gauss_aux_loss(mu, log_std, old_mu, old_std, v, aux, ret, kl_beta):
    """The same for a plain Normal(mu, exp(log_std)) against Normal(old_mu, old_std): KL is [B, D], meaned over B*D."""
    p = Normal(mu, log_std.exp(), validate_args=False)
    q = Normal(old_mu, old_std, validate_args=False)
    aux_loss = F.mse_loss(v.detach(), aux)
    kl_loss = kl_divergence(p, q).mean()
    value_loss = F.mse_loss(v, ret)
    return aux_loss + kl_beta * kl_loss + value_loss, aux_loss, kl_loss, value_loss


def cat_batch(rng, B, A, zeros=True):
    """Logits with the zero-probability regimes: finite logits far enough below the row's max that the probability
    underflows to 0 on the new side (p = 0) and on the old side (q = 0), in float32 and float64 alike."""
    z = rng.normal(size=(B, A)).astype(np.float32) * 2
    o = (z + rng.normal(size=(B, A)).astype(np.float32) * 0.5).astype(np.float32)
    if zeros and A > 1:
        z[0, 0] -= 1e4
        o[min(1, B - 1), A - 1] -= 1e4
        if B > 2:
            z[2, 0] -= 1e4
            o[2, 0] -= 1e4                                          # both 0 on the same term
    v = rng.normal(size=B).astype(np.float32)
    aux = rng.normal(size=B).astype(np.float32)
    ret = rng.normal(size=B).astype(np.float32)
    return z, o, v, aux, ret


def gauss_batch(rng, B, D):
    mu = rng.normal(size=(B, D)).astype(np.float32)
    omu = (mu + rng.normal(size=(B, D)).astype(np.float32) * 0.3).astype(np.float32)
    ls = (rng.normal(size=D) * 0.3 - 0.5).astype(np.float32)
    ols = (ls + rng.normal(size=D) * 0.2).astype(np.float32)
    v = rng.normal(size=B).astype(np.float32)
    aux = rng.normal(size=B).astype(np.float32)
    ret = rng.normal(size=B).astype(np.float32)
    return mu, ls, omu, ols, v, aux, ret


# ---------------------------------------------------------------- the update-cycle fixture (tests/golden/ppg_update.npz)
# Written by tests/golden/make_golden_ppg.py from the unmodified reference: per case, the reference's PhasicActorCritic
# (Basic_MLP, hidden [FIX_HIDDEN], orthogonal init) runs one full cycle of PPG_Learner (POLICY / VALUE / AUX_NEPOCH epochs,
# the relabel between the critic and the auxiliary phases) on FIX_ROWS fixed rows.
FIX_OBS, FIX_HIDDEN, FIX_ROWS, FIX_A, FIX_D = 4, 16, 24, 3, 2
FIX_NEPOCH = {"actor": 2, "critic": 2, "aux": 2}
FIX_LR, FIX_CLIP_NORM, FIX_KL_BETA = 1e-2, 0.05, 1.0
FIX_CASES = [(kind, mb, clip) for kind in ("cat", "gauss") for mb in (1, 2) for clip in (0, 1)]
FIX_INFO_KEYS = {"actor": ["actor-loss", "entropy", "learning_rate", "clip_ratio"], "critic": ["critic-loss"],
                 "aux": ["aux-loss", "kl-loss", "value-loss", "loss"]}


def fix_learner_config(mb, clip):
    """The learner keys of a fixture case (total_iters = 2 * 1 * mb: the LinearLR schedule reaches its end inside it)."""
    return dict(learning_rate=FIX_LR, ent_coef=0.01, clip_range=0.2, kl_beta=FIX_KL_BETA, use_grad_clip=bool(clip),
                grad_clip_norm=FIX_CLIP_NORM, end_factor_lr_decay=0.5, horizon_size=FIX_ROWS, parallels=1,
                running_steps=2 * FIX_ROWS, n_epochs=1, n_minibatch=mb, policy_nepoch=FIX_NEPOCH["actor"],
                value_nepoch=FIX_NEPOCH["critic"], aux_nepoch=FIX_NEPOCH["aux"])


def fix_rows(kind, seed):
    rng = np.random.default_rng(seed)
    obs = rng.normal(size=(FIX_ROWS, FIX_OBS)).astype(np.float32)
    act = (rng.normal(size=(FIX_ROWS, FIX_D)).astype(np.float32) if kind == "gauss"
           else rng.integers(0, FIX_A, FIX_ROWS).astype(np.float32))
    adv = rng.normal(size=FIX_ROWS).astype(np.float32)
    ret = rng.normal(size=FIX_ROWS).astype(np.float32)
    return obs, act, adv, ret


def fix_case_seed(kind, mb, clip):
    return 300 + 10 * (kind == "gauss") + 2 * mb + clip

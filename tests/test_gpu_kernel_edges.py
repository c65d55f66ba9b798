"""GPU: the small fused kernels (K3 scalar gather + advantage normalisation, K4 PPO loss, K6 DQN TD, K7 norm / Adam / soft
update, K8 SAC, K9 QMIX select / mix / TD) called through the C-ABI against the float64 references of tests/kernel_refs.py,
at the shapes and inputs where such kernels go wrong: every template tier, 1 / 255 / 256 / 257 rows and the grid-stride
regime above XB_MAX_PARTIALS * 256 rows, ties, masks, misaligned operands, tails of the float4 loops, and the sharded
minibatch contract of DESIGN.md section 5 emulated on one GPU.

Tolerances.  EPS = 2^-24 is float32's unit roundoff.  A float32 result of k roundings is within k*EPS of the exact result
RELATIVE TO THE MAGNITUDE OF WHAT WAS ADDED (not of the result, which may cancel); each check below builds that magnitude
from the float64 reference and states k.  The logged statistics are summed in float64 and rounded once, so they are held
to the same per-row bound summed over the rows plus 2 EPS of the statistic.  Where the header claims float32 operation
order, results are compared bit for bit."""
import numpy as np
import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = kr.EPS32
f32 = np.float32


def _lib():
    from xuance_b200 import _lib
    return _lib


def _big_rows():
    """First row count in the grid-stride regime: the reductions cap their grid at XB_MAX_PARTIALS blocks of 256 threads,
    and the scratch holds 8 slots of XB_MAX_PARTIALS doubles plus 8."""
    max_partials = (_lib().load().xb_scratch_doubles() - 8) // 8
    return max_partials * 256 + 257


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _within(got, want, tol, what):
    got = np.asarray(got.cpu().numpy() if torch.is_tensor(got) else got, np.float64)
    want, tol = np.broadcast_to(np.asarray(want, np.float64), got.shape), np.broadcast_to(tol, got.shape)
    err = np.abs(got - want)
    bad = ~(err <= tol)                       # NaN (an unwritten output) fails too
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, np.nan_to_num(err / np.maximum(tol, 1e-300), nan=np.inf), 0)), got.shape)
        raise AssertionError(f"{what}: {bad.sum()} of {bad.size} outside tolerance; at {i}: got {got[i]!r} want {want[i]!r} "
                             f"tol {tol[i]!r}")


def _ptrs(*ts):
    return [_lib().ptr(t) for t in ts]


# ====================================================================================================== K4
def _ppo_inputs(B, A, seed):
    """Logits with a +-30 spread, ratios on both sides of 1 -+ clip (never within 1e-2 of a bound, so float32 and float64
    agree on the side), ratio 1, adv = 0 and negative adv."""
    rng = np.random.default_rng(seed)
    logits = rng.uniform(-30, 30, (B, A)).astype(f32)
    act = rng.integers(0, A, B).astype(f32)
    lp = kr._log_softmax(logits)[np.arange(B), act.astype(np.int64)]
    kind = rng.integers(0, 4, B)
    ratio = np.select([kind == 0, kind == 1, kind == 2], [rng.uniform(0.3, 0.79, B), rng.uniform(0.81, 1.19, B),
                                                          rng.uniform(1.21, 3.0, B)], 1.0)
    adv = rng.normal(size=B).astype(f32)
    adv[rng.random(B) < 0.1] = 0.0
    return dict(logits=logits, value=rng.normal(size=B).astype(f32), actions=act,
                old_logp=(lp - np.log(ratio)).astype(f32), adv=adv, ret=rng.normal(size=B).astype(f32))


PPO_HP = dict(clip=0.2, vf_coef=0.25, ent_coef=0.01)


def _run_ppo(x, lo, hi, B_total, kind, scratch):
    B, A = hi - lo, x["logits"].shape[1]
    t = {k: _t(v[lo:hi]) for k, v in x.items()}
    dz, dv, st = _nan(B, A), _nan(B), _nan(8)
    _lib().call("xb_ppo_loss_fwd_bwd", *_ptrs(t["logits"], t["value"], t["actions"], t["old_logp"], t["adv"], t["ret"]), B,
                A, B_total, PPO_HP["clip"], PPO_HP["vf_coef"], PPO_HP["ent_coef"], kind, *_ptrs(dz, dv, st, scratch))
    return dz, dv, st


def _ppo_ref_and_tol(x, B_total, kind):
    """Reference and tolerances.  logp_i = z_i - lse carries an absolute error of a few EPS * c, c = max|z| + |lse| per
    row, so p_i, ratio and every product of them carry a RELATIVE error of a few EPS * c; the entropy adds A roundings.  With
    k = 8 (c + A) the gradient tolerance is k EPS * (|d_logp| (1{i=a} + p_i) + |dent| p_i (|lp_i| + H + 1))."""
    dz, dv, st = kr.ppo_loss(x["logits"], x["value"], x["actions"], x["old_logp"], x["adv"], x["ret"], B_total,
                             f32(PPO_HP["clip"]), f32(PPO_HP["vf_coef"]), f32(PPO_HP["ent_coef"]), kind)
    lp = kr._log_softmax(x["logits"])
    p = np.exp(lp)
    B, A = lp.shape
    a = x["actions"].astype(np.int64)
    H = -(p * lp).sum(1)
    c = np.abs(x["logits"]).max(1) + np.abs(lp[:, 0] - x["logits"][:, 0]) + A
    ratio = np.exp(lp[np.arange(B), a] - x["old_logp"]) if kind == 0 else np.ones(B)
    d_logp = np.abs(x["adv"]) * np.maximum(ratio, 1.0) / B_total
    onehot = np.zeros((B, A))
    onehot[np.arange(B), a] = 1
    k = 8 * c[:, None] * EPS
    tol_dz = k * (d_logp[:, None] * (onehot + p) + PPO_HP["ent_coef"] / B_total * p * (np.abs(lp) + H[:, None] + 1))
    v, r = x["value"].astype(np.float64), x["ret"].astype(np.float64)
    tol_dv = 4 * EPS * PPO_HP["vf_coef"] * 2 * (np.abs(v) + np.abs(r)) / B_total
    smin_mag = np.abs(x["adv"]) * np.maximum(ratio, 1.0 + PPO_HP["clip"]) * np.maximum(np.abs(lp[np.arange(B), a]), 1)
    t_a = (8 * c * EPS * smin_mag).sum() / B_total
    t_c = 4 * EPS * ((v - r) ** 2).sum() / B_total
    t_e = (8 * c * EPS * ((p * np.abs(lp)).sum(1) + 1)).sum() / B_total
    t_v = 2 * EPS * np.abs(v).sum() / B_total
    tol_st = np.array([t_a, t_c, t_e, t_v, 0.0, t_a + PPO_HP["ent_coef"] * t_e + PPO_HP["vf_coef"] * t_c])
    tol_st += 4 * EPS * (np.abs(st) + np.abs(st[0]) + np.abs(st[2]) * PPO_HP["ent_coef"] + np.abs(st[1]))
    return (dz, dv, st), (tol_dz, tol_dv, tol_st)


def _check_ppo(out, x, B_total, kind, what=""):
    (dz, dv, st), (tz, tv, ts) = _ppo_ref_and_tol(x, B_total, kind)
    _within(out[0], dz, tz, what + "dlogits")
    _within(out[1], dv, tv, what + "dvalue")
    got = out[2].cpu().numpy().astype(np.float64)
    _within(got[:6], st, ts, what + "stats")
    assert round(got[4] * B_total) == round(st[4] * B_total), what + "clip fraction counts a different number of rows"
    assert got[6] == 0 and got[7] == 0


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("A", [1, 3, 4, 5, 8, 9, 18, 19, 32, 33, 64])
def test_ppo_loss_tiers_and_row_counts(A, kind):
    scratch = _lib().scratch(DEV)
    sizes = [1, 255, 256, 257] + ([_big_rows()] if A in (1, 3, 4) else [])   # A <= 4: the two-rows-in-flight loop
    for B in sizes:
        x = _ppo_inputs(B, A, seed=B * 100 + A)
        _check_ppo(_run_ppo(x, 0, B, B, kind, scratch), x, B, kind, f"A={A} B={B} kind={kind}: ")


# ====================================================================================================== K6
def _dqn_inputs(B, A, seed):
    rng = np.random.default_rng(seed)
    return dict(q_eval=rng.normal(size=(B, A)).astype(f32), q_next=rng.normal(size=(B, A)).astype(f32),
                q_sel=rng.integers(0, 3, size=(B, A)).astype(f32),      # duplicated maxima: the first index must win
                actions=rng.integers(0, A, B).astype(f32), rew=rng.normal(size=B).astype(f32),
                term=(rng.random(B) < 0.3).astype(f32))


def _run_dqn(x, lo, hi, B_total, double_q, scratch):
    B, A = hi - lo, x["q_eval"].shape[1]
    t = {k: _t(v[lo:hi]) for k, v in x.items()}
    dq, td, st = _nan(B, A), _nan(B), _nan(4)
    _lib().call("xb_dqn_td_fwd_bwd", *_ptrs(t["q_eval"], t["q_next"], t["q_sel"] if double_q else None, t["actions"],
                                            t["rew"], t["term"]), B, A, B_total, 0.99, *_ptrs(dq, td, st, scratch))
    return dq, td, st


def _check_dqn(out, x, B_total, double_q, what=""):
    """td is bit-exact (float32 in torch's order).  |td - exact| <= 3 EPS (|r| + |gamma max| + |pred|) = e, so dq at the
    taken action is within 2 e / B_total + 2 EPS |dq| and exactly 0 elsewhere; loss within sum 2 |td| e / B_total."""
    dq, td32, td, st = kr.dqn_td(x["q_eval"], x["q_next"], x["q_sel"] if double_q else None, x["actions"], x["rew"],
                                 x["term"], B_total, 0.99)
    assert np.array_equal(out[1].cpu().numpy(), td32), what + "td differs from the float32 restatement"
    B = td.shape[0]
    a = x["actions"].astype(np.int64)
    pred = x["q_eval"][np.arange(B), a].astype(np.float64)
    e = 3 * EPS * (np.abs(x["rew"]) + np.abs(td + pred - x["rew"]) + np.abs(pred))
    tol = np.zeros_like(dq)
    tol[np.arange(B), a] = 2 * e / B_total + 2 * EPS * np.abs(dq[np.arange(B), a])
    _within(out[0], dq, tol, what + "dq")
    got = out[2].cpu().numpy()
    _within(got[:2], st, [(2 * np.abs(td) * e).sum() / B_total + 2 * EPS * st[0],
                          2 * EPS * (np.abs(st[1]) + np.abs(pred).sum() / B_total)], what + "stats")
    assert got[2] == 0 and got[3] == 0


@pytest.mark.parametrize("double_q", [False, True])
@pytest.mark.parametrize("A", [1, 2, 6, 18])
def test_dqn_td_ties_and_row_counts(A, double_q):
    scratch = _lib().scratch(DEV)
    for B in [1, 257] + ([_big_rows()] if A == 6 else []):
        x = _dqn_inputs(B, A, seed=B + A)
        _check_dqn(_run_dqn(x, 0, B, B, double_q, scratch), x, B, double_q, f"A={A} B={B} double_q={double_q}: ")


# ====================================================================================================== K8
ALPHA, SAC_GAMMA = f32(0.37), 0.99


def _sac_inputs(B, seed):
    rng = np.random.default_rng(seed)
    x = {k: (rng.normal(size=B) * s).astype(f32) for k, s in
         dict(log_pi=2, q1=3, q2=3, aq1=3, aq2=3, target_q=3, log_pi_next=2, rew=1).items()}
    x["q2"][::3] = x["q1"][::3]                                # torch.min ties: each side gets half
    x["term"] = (rng.random(B) < 0.3).astype(f32)
    return x


def _run_sac(x, lo, hi, B_total, scratch):
    B = hi - lo
    t = {k: _t(v[lo:hi]) for k, v in x.items()}
    alpha = _t(np.array([ALPHA]))                              # the temperature lives in device memory
    a_out, c_out = [_nan(B) for _ in range(3)] + [_nan(4)], [_nan(B) for _ in range(3)] + [_nan(2)]
    _lib().call("xb_sac_actor_loss", *_ptrs(t["log_pi"], t["q1"], t["q2"], alpha), B, B_total, *_ptrs(*a_out, scratch))
    _lib().call("xb_sac_critic_loss", *_ptrs(t["aq1"], t["aq2"], t["target_q"], t["log_pi_next"], t["rew"], t["term"], alpha),
                SAC_GAMMA, B, B_total, *_ptrs(*c_out, scratch))
    return a_out, c_out


def _check_sac(out, x, B_total, what=""):
    """Actor: the seeds are one or two roundings of exact values (2 EPS relative); Ploss adds fl(alpha*lp) - min per row (2
    EPS of |alpha lp| + |min q|).  Critic: backup is bit-exact; e = q - backup is within EPS |e| + 3 EPS (|r| + |target|
    + |alpha lp'|) = d, so dq within 2 d / B_total + 2 EPS |dq|, Qloss within sum 2 |e| d / B_total per critic."""
    (dlp, dq1, dq2, st), (a_out, c_out) = kr.sac_actor(x["log_pi"], x["q1"], x["q2"], ALPHA, B_total), out
    _within(a_out[0], dlp, 2 * EPS * np.abs(dlp), what + "dlog_pi")
    _within(a_out[1], dq1, EPS * np.abs(dq1), what + "dq1 (actor)")
    _within(a_out[2], dq2, EPS * np.abs(dq2), what + "dq2 (actor)")
    lp, mq = x["log_pi"].astype(np.float64), np.minimum(x["q1"], x["q2"]).astype(np.float64)
    got = a_out[3].cpu().numpy()
    _within(got[:3], st, [2 * EPS * (np.abs(ALPHA * lp) + np.abs(mq)).sum() / B_total + 2 * EPS * abs(st[0]),
                          2 * EPS * np.abs(mq).sum() / B_total, 2 * EPS * np.abs(lp).sum() / B_total], what + "actor stats")
    assert got[3] == 0
    cq1, cq2, y, cst = kr.sac_critic(x["aq1"], x["aq2"], x["target_q"], x["log_pi_next"], x["rew"], x["term"], ALPHA,
                                     SAC_GAMMA, B_total)
    assert np.array_equal(c_out[2].cpu().numpy(), kr.sac_backup_f32(x["target_q"], x["log_pi_next"], x["rew"], x["term"],
                                                                      ALPHA, SAC_GAMMA)), what + "backup"
    d0 = 3 * EPS * (np.abs(x["rew"]) + np.abs(x["target_q"]) + np.abs(ALPHA * x["log_pi_next"]))
    qloss_tol = 4 * EPS * cst[0]
    for q, g, ref in ((x["aq1"], c_out[0], cq1), (x["aq2"], c_out[1], cq2)):
        e = q - y
        d = EPS * np.abs(e) + d0
        _within(g, ref, 2 * d / B_total + 2 * EPS * np.abs(ref), what + "dq (critic)")
        qloss_tol += (2 * np.abs(e) * d).sum() / B_total
    _within(c_out[3].cpu().numpy()[:1], cst, qloss_tol, what + "Qloss")
    assert c_out[3][1].item() == 0


def test_sac_losses_ties_device_alpha_and_row_counts():
    scratch = _lib().scratch(DEV)
    for B in (1, 257, _big_rows()):
        x = _sac_inputs(B, seed=B)
        _check_sac(_run_sac(x, 0, B, B, scratch), x, B, f"B={B}: ")


# ====================================================================================================== K9 select
@pytest.mark.parametrize("double_q", [0, 1])
@pytest.mark.parametrize("with_avail", [False, True])
@pytest.mark.parametrize("B,n,T,A", [(3, 5, 7, 6), (64, 9, 40, 12)])
def test_qmix_select_masks_ties_and_availability(B, n, T, A, with_avail, double_q):
    """Values and masks in {0, 1} make every output exact: the gathers, arg-max and max are compared bit for bit."""
    rng = np.random.default_rng(B * n + double_q)
    q_all = rng.integers(-2, 3, size=(B, n, T + 1, A)).astype(f32)              # ties in the double-Q arg-max
    q_tgt = rng.normal(size=(B, n, T + 1, A)).astype(f32)
    actions = rng.integers(0, A, size=(B, n, T)).astype(f32)
    agent_mask = (rng.random((B, n, T)) < 0.8).astype(f32)
    filled = (rng.random((B, T)) < 0.8).astype(f32)
    ld = A + 3                                                                  # avail rows longer than A
    avail = (rng.random((B, n, T + 1, ld)) < 0.6).astype(np.uint8)
    avail[0, 0, 2, :A] = 0                                                      # a step with no action available
    agent_mask[0, 0, 1] = filled[0, 1] = 1.0                                   # ... whose next value is used
    t = [_t(v) for v in (q_all, q_tgt, actions, agent_mask, filled)]
    av = _t(avail) if with_avail else None
    qe, qn, fs = _nan(B * T, n), _nan(B * T, n), _nan(1)
    L = _lib()
    scratch = L.scratch(DEV)
    L.call("xb_qmix_select_fwd", *_ptrs(*t, av), ld if with_avail else 0, B, n, T, A, double_q, *_ptrs(qe, qn, fs, scratch))
    ref = kr.qmix_select(q_all, q_tgt, actions, agent_mask, filled, avail if with_avail else None, double_q)
    assert np.array_equal(qe.cpu().numpy(), ref[0])
    assert np.array_equal(qn.cpu().numpy(), ref[1])
    assert fs.item() == ref[2]
    d = rng.normal(size=(B * T, n)).astype(f32)
    dq_all = torch.zeros((B, n, T + 1, A), device=DEV)
    dd = _t(d)
    L.call("xb_qmix_select_bwd", *_ptrs(dd, t[2], t[3], t[4]), B, n, T, A, L.ptr(dq_all))
    assert np.array_equal(dq_all.cpu().numpy(), kr.qmix_select_bwd(d, actions, agent_mask, filled, A))


# ====================================================================================================== K9 mix
@pytest.mark.parametrize("R", [1, 3, 777])
@pytest.mark.parametrize("H", [32, 48, 64])
@pytest.mark.parametrize("n", [1, 5, 9, 16])
def test_qmix_mix_forward_backward(n, H, R):
    """Float64 autograd of elu(q |w1| + b1) |w2| + b2.  With u_j = 1 + |b1_j| + sum_i |q_i w1_ij| (the magnitude of the
    pre-activation's summands), pre_j carries (n+1) EPS u_j, elu' = exp(pre) = h + 1 an absolute (n+4) EPS u_j, and the
    H-term sums (H/32 per lane, then a 5-level shuffle tree) H/32 + 6 more roundings, so every output is held to
    k EPS * (its summands' magnitudes, each scaled by u_j) with k = n + H/32 + 12."""
    rng = np.random.default_rng(n * 1000 + H + R)
    q = (rng.normal(size=(R, n)) * 2).astype(f32)
    w1 = (rng.normal(size=(R, n * H)) / np.sqrt(n)).astype(f32)
    b1 = rng.normal(size=(R, H)).astype(f32)
    w2 = (rng.normal(size=(R, H)) / np.sqrt(H)).astype(f32)
    b2, g = rng.normal(size=(2, R)).astype(f32)
    q_tot, dq, dw1, db1, dw2 = kr.qmix_mix(q, w1, b1, w2, b2, g, n, H)
    u = 1 + np.abs(b1) + np.einsum("ri,rij->rj", np.abs(q), np.abs(w1.reshape(R, n, H)))
    k = (n + H // 32 + 12) * EPS
    aw1, aw2, ag = np.abs(w1.reshape(R, n, H)), np.abs(w2), np.abs(g)[:, None]
    tols = (k * ((aw2 * u).sum(1) + np.abs(b2)), k * np.einsum("rj,rij->ri", ag * aw2 * u, aw1),
            (k * (ag * aw2 * u)[:, None, :] * np.abs(q)[:, :, None]).reshape(R, n * H), k * ag * aw2 * u, k * ag * u)
    L = _lib()
    for offset in ((0, 1) if H == 32 else (0,)):    # w1 one float into a larger buffer: H = 32 takes the generic kernel
        w1_buf = torch.zeros(R * n * H + 1, device=DEV)
        w1_buf[offset:offset + R * n * H] = _t(w1.reshape(-1))
        w1_d = w1_buf[offset:offset + R * n * H]
        tq, tb1, tw2, tb2, tg = (_t(v) for v in (q, b1, w2, b2, g))
        outs = (_nan(R), _nan(R, n), _nan(R, n * H), _nan(R, H), _nan(R, H))
        L.call("xb_qmix_mix_fwd", *_ptrs(tq, w1_d, tb1, tw2, tb2), R, n, H, L.ptr(outs[0]))
        L.call("xb_qmix_mix_bwd", *_ptrs(tg, tq, w1_d, tb1, tw2), R, n, H, *_ptrs(*outs[1:]))
        for name, got, want, tol in zip(("q_tot", "dq", "dw1", "db1", "dw2"), outs, (q_tot, dq, dw1, db1, dw2), tols):
            _within(got, want, tol, f"n={n} H={H} R={R} w1 offset {offset}: {name}")


# ====================================================================================================== K9 TD
def _qmix_td_inputs(B, n, T, seed):
    rng = np.random.default_rng(seed)
    term = rng.random((B, n, T)) < 0.5
    term[:, :, T - 1] = rng.random((B, 1)) < 0.5                  # whole-team terminals at the last step
    filled = np.ones((B, T), f32)
    for b in range(B):
        filled[b, rng.integers(1, T + 1):] = 0.0                   # padded tails of shorter episodes
    return dict(q_tot=(rng.normal(size=B * T) * 3).astype(f32), q_tot_next=(rng.normal(size=B * T) * 3).astype(f32),
                rewards=rng.normal(size=(B, n, T)).astype(f32), terminals=term.astype(f32), filled=filled)


def _run_qmix_td(x, lo, hi, rows_total, filled_sum, scratch):
    """Episodes lo..hi of the batch; filled_sum (float) and rows_total are the global values."""
    B, n, T = hi - lo, x["rewards"].shape[1], x["rewards"].shape[2]
    t = [_t(x["q_tot"][lo * T:hi * T]), _t(x["q_tot_next"][lo * T:hi * T]), _t(x["rewards"][lo:hi]),
         _t(x["terminals"][lo:hi]), _t(x["filled"][lo:hi]), _t(np.array([filled_sum], f32))]
    dq, st = _nan(B * T), _nan(2)
    _lib().call("xb_qmix_td", *_ptrs(*t), B, n, T, 0.99, rows_total, *_ptrs(dq, st, scratch))
    return dq, st


def _check_qmix_td(out, x, what=""):
    """td = (q - y) f with y = mean_i r_i + (1-d) gamma q' is within e = (n+5) EPS (|q| + mean_i |r_i| + |gamma q'|);
    dq within 2 f e / sum(f) + 3 EPS |dq| (exactly 0 where f = 0), loss within sum 2 |td| e / sum(f), predictQ 2 EPS."""
    B, n, T = x["rewards"].shape
    fs = float(x["filled"].sum())
    dq, st = kr.qmix_td(x["q_tot"], x["q_tot_next"], x["rewards"], x["terminals"], x["filled"], fs, 0.99, B * T)
    f = x["filled"].reshape(-1)
    e = (n + 5) * EPS * (np.abs(x["q_tot"]) + np.abs(x["rewards"]).mean(1).reshape(-1) + np.abs(0.99 * x["q_tot_next"]))
    _within(out[0], dq, 2 * f * e / fs + 3 * EPS * np.abs(dq), what + "dq_tot")
    td = np.abs(dq) * fs / 2
    _within(out[1], st, [(2 * td * e).sum() / fs + 2 * EPS * st[0], 2 * EPS * (np.abs(st[1]) + np.abs(x["q_tot"]).sum()
                                                                                / (B * T))], what + "stats")


def test_qmix_td_team_reward_terminal_and_padding():
    x = _qmix_td_inputs(24, 5, 13, seed=9)
    x["terminals"][0, :, 3] = 1.0                                  # every agent terminal: team terminal
    x["terminals"][1, :4, 3], x["terminals"][1, 4, 3] = 1.0, 0.0   # one agent alive: not terminal
    B, n, T = x["rewards"].shape
    out = _run_qmix_td(x, 0, B, B * T, float(x["filled"].sum()), _lib().scratch(DEV))
    _check_qmix_td(out, x)
    assert (out[0].cpu().numpy()[x["filled"].reshape(-1) == 0] == 0).all()


# ====================================================================================================== K7
@pytest.mark.parametrize("n", [1, 2, 3, 5, 1023, (1 << 22) + 3])
def test_grad_sumsq_tails(n):
    """sqrt(sum g^2) * grad_scale: squares and sums in float64, one float32 rounding of the result (2 EPS with the
    float32 grad_scale)."""
    g = np.random.default_rng(n).normal(size=n).astype(f32)
    gd, out, scratch = _t(g), _nan(1), _lib().scratch(DEV)      # named: a temporary's memory may be reused before the launch
    _lib().call("xb_grad_sumsq", *_ptrs(gd), n, 0.75, *_ptrs(out, scratch))
    want = kr.grad_norm(g, 0.75)
    _within(out, [want], 2 * EPS * want, f"n={n}")


@pytest.mark.parametrize("write_back", [0, 1])
@pytest.mark.parametrize("clip", ["active", "inactive", "zero", "negative"])
@pytest.mark.parametrize("n", [3, 4099])
def test_adam_step_against_float64_and_torch(n, clip, write_back):
    """Three steps of xb_adam_step after xb_grad_sumsq, grad_scale 0.5.  Against the float64 Adam rule: the clip factor
    carries 4 EPS (norm, max_norm, division, product), g'^2 twice that, and m, v, the square root, the division and the
    product a few roundings more, so each step's update step_size m / (sqrt(v)/bc2 + eps) is within 32 t EPS of its
    magnitude at step t and p adds 2 EPS |p| per step; m and v are held to 16 t EPS of their summands.  Against
    torch.optim.Adam on the CPU fed the same clipped float32 gradient: the kernel's weights 1 - b1 and 1 - b2 are float32
    differences of the float32 betas, torch's are the float32 roundings of the double differences; they differ by d1 and d2
    relative (1.3e-5 for b2 = 0.999), so the update differs by t (d1 + d2/2) of its size on top of the roundings."""
    L = _lib()
    rng = np.random.default_rng(n)
    b1, b2, eps, lr, scale = 0.9, 0.999, 1e-5, 1e-3, 0.5
    p0 = rng.normal(size=n).astype(f32)
    p, m, v = _t(p0), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    hyper, norm, scratch = torch.zeros(4, device=DEV), _nan(1), L.scratch(DEV)
    tp = torch.tensor(p0, requires_grad=True)
    opt = torch.optim.Adam([tp], lr=lr, betas=(b1, b2), eps=eps)
    rp, rm, rv, mm = p0.astype(np.float64), np.zeros(n), np.zeros(n), np.zeros(n)
    tol_p, tol_torch = np.zeros(n), np.zeros(n)
    w32 = lambda b: (f32(1) - f32(b), f32(1 - b))
    d1, d2 = (abs(float(a) - float(b)) / float(b) for a, b in (w32(b1), w32(b2)))
    for t in range(1, 4):
        g = (rng.normal(size=n) * 1e-2).astype(f32)
        g[::5] *= 1e-5                                           # |g| near eps: the eps regime of the denominator
        gd = _t(g)
        hyper.copy_(torch.tensor([lr / (1 - b1 ** t), np.sqrt(1 - b2 ** t), lr, 0.0]))
        L.call("xb_grad_sumsq", L.ptr(gd), n, scale, L.ptr(norm), L.ptr(scratch))
        true_norm = kr.grad_norm(g, scale)
        max_norm = {"active": 0.5 * true_norm, "inactive": 10 * true_norm, "zero": 0.0, "negative": -1.0}[clip]
        L.call("xb_adam_step", *_ptrs(p, gd, m, v), n, L.ptr(hyper), b1, b2, eps, max_norm, L.ptr(norm), scale, write_back)
        # the gradient the kernel applies, float32 restated from its norm
        nf = f32(norm.item())
        c = f32(scale) * min(f32(max_norm) / (nf + f32(1e-6)), f32(1)) if max_norm > 0 else f32(scale)
        g_used = g * c
        assert np.array_equal(gd.cpu().numpy(), g_used if write_back else g), "gradient write-back"
        hp = hyper.cpu().numpy()
        rp_new, _, rm, rv = kr.adam_step(rp, g, rm, rv, hp[0], hp[1], b1, b2, eps, kr.adam_coef(true_norm, max_norm, scale))
        mm = b1 * mm + (1 - b1) * np.abs(g_used)
        tol_p += 2 * EPS * np.abs(rp) + 32 * t * EPS * np.abs(rp_new - rp)
        tol_torch += (t * (d1 + d2 / 2) + 32 * t * EPS) * np.abs(rp_new - rp)
        rp = rp_new
        _within(p, rp, tol_p, f"step {t}: p")
        _within(m, rm, 16 * t * EPS * mm, f"step {t}: m")
        _within(v, rv, 16 * t * EPS * rv, f"step {t}: v")
        tp.grad = torch.from_numpy(g_used)
        opt.step()
        _within(p, tp.detach().numpy(), 4 * EPS * np.abs(rp) + tol_torch, f"step {t}: p vs torch")


def test_soft_update_is_bit_exact():
    rng = np.random.default_rng(11)
    n = 4099
    tgt, src = (rng.normal(size=(2, n)) * 3).astype(f32)
    t = _t(tgt)
    s = _t(src)
    _lib().call("xb_soft_update", *_ptrs(t, s), n, 0.005)
    assert np.array_equal(t.cpu().numpy(), kr.soft_update_f32(tgt, src, 0.005))


# ====================================================================================================== K3
def test_gather_scalars_statistics_and_normalisation_at_large_batch():
    """mean / population std over more than XB_MAX_PARTIALS * 256 gathered rows: float64 sums, one float32 rounding (2 EPS;
    the std's E[x^2] - mean^2 cancels by less than a factor 2 here).  The normalisation given those statistics is
    bit-exact, and so is xb_adv_normalize alone."""
    L = _lib()
    rng = np.random.default_rng(12)
    B, F, slots = _big_rows(), 3, 600_000
    fields = (rng.normal(size=(F, slots)) + 0.3).astype(f32)
    idx = rng.permutation(slots)[:B].astype(np.int64)
    fd, idx_d, out, stats, scratch = _t(fields), _t(idx), _nan(F, B), _nan(2), L.scratch(DEV)
    L.call("xb_gather_scalars", L.ptr(fd), slots, L.ptr(idx_d), B, F, L.ptr(out), 1, *_ptrs(stats, scratch))
    got = out.cpu().numpy()
    assert np.array_equal(got[0], fields[0, idx]) and np.array_equal(got[2], fields[2, idx])
    mean, std = kr.adv_stats(fields[1, idx])
    st = stats.cpu().numpy()
    _within(st, [mean, std], [2 * EPS * abs(mean), 4 * EPS * std], "statistics")
    assert np.array_equal(got[1], kr.adv_normalize_f32(fields[1, idx], st))
    for n in (1, B):
        a = fields[2, :n].copy()
        given = np.array([0.25, 1.75], f32)
        ad, gd = _t(a), _t(given)
        L.call("xb_adv_normalize", L.ptr(ad), n, L.ptr(gd))
        assert np.array_equal(ad.cpu().numpy(), kr.adv_normalize_f32(a, given))


# ====================================================================================================== sharded minibatches
def _shards(B, G):
    s = B // G
    return [(g * s, (g + 1) * s) for g in range(G)]


def _sum_stats(parts, whole, what):
    """The all-reduce sums the ranks' float32 statistics; each part and the unsharded result are rounded once, so the sum
    agrees with the unsharded launch to 2 EPS of the parts' magnitudes (in float64, as the sum is exact there)."""
    parts = np.stack([p.cpu().numpy().astype(np.float64) for p in parts])
    whole = whole.cpu().numpy().astype(np.float64)
    _within(parts.sum(0), whole, 2 * EPS * (np.abs(parts).sum(0) + np.abs(whole)), what)
    return parts.sum(0)


@pytest.mark.parametrize("G", [2, 3, 8])
def test_sharded_minibatch_contract(G):
    """DESIGN.md section 5: every loss kernel divides by the GLOBAL count, so a rank's shard launched with B_total (or the
    all-reduced sum(filled), rows_total) writes the global-minibatch gradient rows bit for bit, and its statistics sum over
    the ranks to the global ones."""
    scratch = _lib().scratch(DEV)
    cat = lambda xs: torch.cat([x.reshape(-1) for x in xs]).cpu().numpy()
    same = lambda parts, whole, what: np.testing.assert_array_equal(cat(parts), whole.reshape(-1).cpu().numpy(), what)
    B = 2400
    x = _ppo_inputs(B, 6, seed=G)
    whole = _run_ppo(x, 0, B, B, 0, scratch)
    parts = [_run_ppo(x, lo, hi, B, 0, scratch) for lo, hi in _shards(B, G)]
    same([p[0] for p in parts], whole[0], "K4 dlogits")
    same([p[1] for p in parts], whole[1], "K4 dvalue")
    summed = _sum_stats([p[2] for p in parts], whole[2], "K4 stats")
    _check_ppo((whole[0], whole[1], torch.from_numpy(summed.astype(f32))), x, B, 0, "K4 summed: ")

    x = _dqn_inputs(B, 5, seed=G)
    whole = _run_dqn(x, 0, B, B, True, scratch)
    parts = [_run_dqn(x, lo, hi, B, True, scratch) for lo, hi in _shards(B, G)]
    same([p[0] for p in parts], whole[0], "K6 dq")
    same([p[1] for p in parts], whole[1], "K6 td")
    summed = _sum_stats([p[2] for p in parts], whole[2], "K6 stats")
    _check_dqn((whole[0], whole[1], torch.from_numpy(summed.astype(f32))), x, B, True, "K6 summed: ")

    x = _sac_inputs(B, seed=G)
    whole = _run_sac(x, 0, B, B, scratch)
    parts = [_run_sac(x, lo, hi, B, scratch) for lo, hi in _shards(B, G)]
    for stage in (0, 1):
        for i in range(3):
            same([p[stage][i] for p in parts], whole[stage][i], f"K8 stage {stage} output {i}")
    summed = [torch.from_numpy(_sum_stats([p[s][3] for p in parts], whole[s][3], f"K8 stats {s}").astype(f32))
              for s in (0, 1)]
    _check_sac(([*whole[0][:3], summed[0]], [*whole[1][:3], summed[1]]), x, B, "K8 summed: ")

    Be, n, T = 24, 5, 13
    x = _qmix_td_inputs(Be, n, T, seed=G)
    fs = float(x["filled"].sum())                                  # the all-reduced sum(filled)
    whole = _run_qmix_td(x, 0, Be, Be * T, fs, scratch)
    parts = [_run_qmix_td(x, lo, hi, Be * T, fs, scratch) for lo, hi in _shards(Be, G)]
    same([p[0] for p in parts], whole[0], "K9 dq_tot")
    summed = _sum_stats([p[1] for p in parts], whole[1], "K9 stats (loss_Q, predictQ)")
    _check_qmix_td((whole[0], torch.from_numpy(summed.astype(f32))), x, "K9 summed: ")

    # K3: the global statistics from the ranks' moments, as global_adv_stats all-reduces them, and the normalisation
    L = _lib()
    a = (np.random.default_rng(G).normal(size=B) * 2 + 0.5).astype(f32)
    ad, out, stats = _t(a), _nan(1, B), _nan(2)
    L.call("xb_gather_scalars", L.ptr(ad), B, None, B, 1, L.ptr(out), 0, *_ptrs(stats, scratch))
    mom = sum(np.array([a[lo:hi].astype(np.float64).sum(), (a[lo:hi].astype(np.float64) ** 2).sum(), hi - lo])
              for lo, hi in _shards(B, G))
    mean = mom[0] / mom[2]
    _within(stats, [mean, np.sqrt(mom[1] / mom[2] - mean * mean)], 4 * EPS * np.abs(stats.cpu().numpy()), "K3 stats")
    shards = [_t(a[lo:hi]) for lo, hi in _shards(B, G)]
    for s in shards:
        L.call("xb_adv_normalize", L.ptr(s), s.numel(), L.ptr(stats))
    same(shards, out, "K3 normalised advantages")


# ====================================================================================================== determinism
def test_grid_reduction_is_deterministic_and_the_shared_scratch_rearms():
    """Three launches at the full 2048-block grid give bit-identical statistics and gradients; then launches of
    different grid sizes interleaved on ONE scratch (its ticket counter re-arms after every reduction) reproduce their
    solo results bit for bit and match their references."""
    B = _big_rows()
    x = _ppo_inputs(B, 4, seed=13)
    runs = [_run_ppo(x, 0, B, B, 0, _lib().scratch(DEV)) for _ in range(3)]
    for r in runs[1:]:
        for a, b in zip(r, runs[0]):
            assert torch.equal(a, b)
    _check_ppo(runs[0], x, B, 0, "full grid: ")

    xs = dict(ppo=_ppo_inputs(257, 7, seed=14), dqn=_dqn_inputs(300, 5, seed=15), sac=_sac_inputs(70_000, seed=16))
    g = np.random.default_rng(17).normal(size=(1 << 20) + 1).astype(f32)
    L = _lib()

    def sumsq(scratch):
        gd, out = _t(g), _nan(1)
        L.call("xb_grad_sumsq", L.ptr(gd), g.size, 1.0, *_ptrs(out, scratch))
        return (out,)

    launches = [lambda s: _run_ppo(x, 0, B, B, 0, s), lambda s: _run_dqn(xs["dqn"], 0, 300, 300, True, s),
                lambda s: [t for stage in _run_sac(xs["sac"], 0, 70_000, 70_000, s) for t in stage], sumsq,
                lambda s: _run_ppo(xs["ppo"], 0, 257, 257, 1, s)]
    solo = [f(_lib().scratch(DEV)) for f in launches]
    shared = L.scratch(DEV)
    for rnd in range(2):
        for f, want in zip(launches, solo):
            for a, b in zip(f(shared), want):
                assert torch.equal(a, b), f"round {rnd}"
    _check_dqn(solo[1], xs["dqn"], 300, True, "interleaved: ")
    _check_sac((solo[2][:4], solo[2][4:]), xs["sac"], 70_000, "interleaved: ")
    _within(solo[3][0], [kr.grad_norm(g, 1.0)], 2 * EPS * kr.grad_norm(g, 1.0), "interleaved: grad norm")
    _check_ppo(solo[4], xs["ppo"], 257, 1, "interleaved: ")

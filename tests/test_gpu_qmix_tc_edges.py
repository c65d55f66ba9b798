"""GPU: K9-TC (xb_qmix_mix_fused_fwd, the tensor-core QMIX mixer forward) against the float64 mixer of tests/qmix_tc_refs.py
at its edge shapes - one agent, the smallest K padding, the largest fusable state for each agent count, tails of a tile and
persistent CTAs whose last tile is unaligned - and bit for bit against itself: a row's value may not depend on the launch,
R, its tile position or how its tile was staged, a NaN stays in its row, and nothing is written past R.

Tolerances are measured on an H100 SXM (80 GB, 700 W power limit) and stated with headroom; each is printed by its test."""
import ctypes

import numpy as np
import pytest
import torch

import qmix_tc_refs as qr
from test_qmix_tc_refs import MAX_RATIO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# max |err| / (KAPPA M_row) over all cases: the bound proves <= 1; the split arithmetic measures about 1e-3 (H100 and the
# CPU model of test_qmix_tc_refs alike), a dropped product 0.3 .. 0.7.  Measured max 1.9e-3 on H100, asserted MAX_RATIO.
# The bias gate: the signed mean of err / (KAPPA M_row) over 2^17 rows must be within 4 standard errors (about 6.5e-7)
# of zero plus BIAS_FLOOR, the residual bias of the hi.hi chain.  Measured -1.5e-5 on H100 with the corrections issued
# first (-3.8e-5 with hi.hi first), asserted |mean| <= 4 se + 2e-5.
BIAS_FLOOR = 2e-5
NS = [1, 2, 5, 8]
RS = [1, 63, 64, 65, 127, 128, 129, 2240]


def _s_max(n):
    """The largest state size QMIX_Mixer._fusable accepts for n agents."""
    from types import SimpleNamespace
    from xuance_b200.torch.rl_models import QMIX_Mixer
    ok = lambda S: QMIX_Mixer._fusable(SimpleNamespace(use_tensor_core_forward=True, dim_hidden=32,
                                                       dim_hypernet_hidden=32, n_agents=n, dim_state=S))
    return max(S for S in range(1, 1024) if ok(S))


def _mixer(S, n, big, seed=0):
    from xuance_b200.torch.rl_models import QMIX_Mixer
    torch.manual_seed(1000 * n + S + seed)
    pm = QMIX_Mixer(S, 32, 32, n, DEV)
    if big:
        with torch.no_grad():
            for k, v in pm.named_parameters():
                if k.endswith("weight"):
                    v.mul_(8.0)
    assert pm._fusable(), (S, n)
    return pm


def _inputs(R, S, n, big, seed=0):
    rng = np.random.default_rng(seed + 7 * S + n)
    if big:
        return rng.uniform(-5, 25, (R, n)).astype(np.float32), rng.uniform(-1, 1, (R, S)).astype(np.float32)
    return (rng.normal(size=(R, n)) * 2).astype(np.float32), rng.normal(size=(R, S)).astype(np.float32)


def _fused(pm, q, st):
    """q_tot [R] through QMIX_Mixer.forward_fused."""
    with torch.no_grad():
        return pm.forward_fused(torch.as_tensor(q, device=DEV), torch.as_tensor(st, device=DEV)).view(-1).cpu().numpy()


def _ratio(pm, q, st, got):
    ref, M = qr.mixer_ref_chunked(qr.mixer_params(pm), q, st)
    return (got.astype(np.float64) - ref) / (qr.KAPPA * M)


def _check(pm, q, st, got, what):
    r = np.abs(_ratio(pm, q, st, got))
    print("K9-TC vs float64 %s: max |err|/(kappa M) %.3g" % (what, r.max()))
    assert np.isfinite(got).all(), what
    assert r.max() <= MAX_RATIO, (what, r.max(), int(r.argmax()))


@pytest.mark.parametrize("big", [False, True], ids=["default-init", "weights-x8"])
@pytest.mark.parametrize("n", NS)
def test_against_float64_and_across_R(n, big):
    """S in {81 (KP1 = 96), 96, 97, 98, the largest fusable S}, every R in RS on prefixes of one input: each launch within
    the bound, and a row's value identical across R (tails of 1, 63, 65, 127 or 129 rows, staged from global memory or
    by the bulk copy depending on rows * S * 4 % 16)."""
    for S in sorted({81, 96, 97, 98, _s_max(n)}):
        pm = _mixer(S, n, big)
        q, st = _inputs(max(RS), S, n, big)
        full = _fused(pm, q, st)
        _check(pm, q, st, full, "n=%d S=%d R=%d" % (n, S, len(q)))
        for R in RS[:-1]:
            got = _fused(pm, q[:R], st[:R])
            assert np.array_equal(got, full[:R]), (n, S, R)


@pytest.mark.parametrize("n,S", [(5, 98), (1, None), (8, None), (2, 97)])
def test_multi_tile_unaligned_last_tile(n, S):
    """R = sm * 256 + t: every CTA runs two full tiles and CTA 0 a third, the tail, whose bulk copy is skipped when
    t * S * 4 is not a multiple of 16 (it is staged from global memory; the mbarrier phase must stay consistent).  Each
    row equals the same row launched alone in chunks that put it at other tile positions, and lies within the bound."""
    S = S or _s_max(n)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    tails = [t for t in range(1, 128) if (t * S * 4) % 16 == 0][:1] + [t for t in range(1, 128) if (t * S * 4) % 16][:1]
    pm = _mixer(S, n, False, seed=1)
    for t in tails:
        R = sm * 256 + t
        q, st = _inputs(R, S, n, False, seed=t)
        full = _fused(pm, q, st)
        _check(pm, q, st, full, "n=%d S=%d R=%d (tail %d)" % (n, S, R, t))
        for step in (1000, 64 * 5 + 1):        # tile positions shifted by 1000 % 128 and 65 rows
            parts = np.concatenate([_fused(pm, q[i:i + step], st[i:i + step]) for i in range(0, R, step)])
            assert np.array_equal(parts, full), (t, step, int(np.flatnonzero(parts != full)[0]))
        again = _fused(pm, q, st)
        assert np.array_equal(again, full)


def test_nan_stays_in_its_row():
    """A NaN in one row's state and another row's q: only those rows are NaN, every other row is bit-identical to the
    clean launch - rows in the same warp, the other warpgroup, the next tile and the unaligned tail tile."""
    n, S, R = 5, 98, 3 * 128 + 37
    pm = _mixer(S, n, False)
    q, st = _inputs(R, S, n, False)
    clean = _fused(pm, q, st)
    for rows_st, rows_q in (([5], [70]), ([130], [200]), ([3 * 128 + 10], [3 * 128 + 36]), ([0], [127])):
        q2, st2 = q.copy(), st.copy()
        for r in rows_st:
            st2[r, S // 2] = np.nan
        for r in rows_q:
            q2[r, n - 1] = np.nan
        got = _fused(pm, q2, st2)
        bad = sorted(rows_st + rows_q)
        assert np.flatnonzero(np.isnan(got)).tolist() == bad, (bad, np.flatnonzero(np.isnan(got)).tolist())
        keep = np.ones(R, bool)
        keep[bad] = False
        assert np.array_equal(got[keep], clean[keep])


@pytest.mark.parametrize("R", [1, 65, 128, 129, 2240])
def test_nothing_written_past_R(R):
    """Sentinels after q_tot[R-1] in the output allocation are untouched (the same ABI call forward_fused makes)."""
    from xuance_b200 import _lib
    n, S = 5, 97                       # 97 * 4 bytes per row: tails of 1 and 65 rows are staged from global memory
    pm = _mixer(S, n, False)
    q, st = _inputs(R, S, n, False)
    qd, sd = torch.as_tensor(q, device=DEV), torch.as_tensor(st, device=DEV)
    pad = 4096
    out = torch.full((R + pad,), 12345.0, device=DEV)
    l1 = [pm.hyper_w_1[0], pm.hyper_b_1, pm.hyper_w_2[0], pm.hyper_b_2[0]]
    w_ptrs = (ctypes.c_void_p * 4)(*[_lib.ptr(m.weight) for m in l1])
    b_ptrs = (ctypes.c_void_p * 4)(*[_lib.ptr(m.bias) for m in l1])
    l2 = [pm.hyper_w_1[2].weight, pm.hyper_w_1[2].bias, pm.hyper_w_2[2].weight, pm.hyper_w_2[2].bias,
          pm.hyper_b_2[2].weight, pm.hyper_b_2[2].bias]
    _lib.call("xb_qmix_mix_fused_fwd", _lib.ptr(sd), _lib.ptr(qd), w_ptrs, b_ptrs, *[_lib.ptr(t) for t in l2], R, S, n,
              32, 32, _lib.ptr(out))
    o = out.cpu().numpy()
    assert (o[R:] == np.float32(12345.0)).all()
    assert np.array_equal(o[:R], _fused(pm, q, st))


def test_bias_gate():
    """Over 2^17 + 37 rows of the 5m_vs_6m shape (n = 5, S = 98) at default initialisation, the signed error in units of
    the bound has a mean within 4 standard errors of zero plus BIAS_FLOOR: the truncating fp32 accumulation of the tensor
    core must not add up to a systematic shift of q_tot."""
    n, S, R = 5, 98, 2 ** 17 + 37
    pm = _mixer(S, n, False, seed=2)
    q, st = _inputs(R, S, n, False, seed=2)
    t = _ratio(pm, q, st, _fused(pm, q, st))
    mean, sd = t.mean(), t.std()
    se = sd / np.sqrt(R)
    print("K9-TC bias gate (units of kappa M_row): max |err| %.3g, mean %.3g, sd %.3g, 4 se + floor %.3g"
          % (np.abs(t).max(), mean, sd, 4 * se + BIAS_FLOOR))
    assert np.abs(t).max() <= MAX_RATIO
    assert abs(mean) <= 4 * se + BIAS_FLOOR, (mean, se)


def test_learner_target_mixer_within_bound():
    """In QMIX_Learner.update after a target sync, Qtarget_tot through K9-TC and through the cuBLAS + K9 path
    (use_tensor_core_forward = False) both lie within the bound of the float64 mixer of the same inputs."""
    from argparse import Namespace
    from helpers import qmix_episode_stream
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners.qmix_learner import QMIX_Learner
    from test_gpu_qmix import _product_model, _buffers
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(3)
    n, obs_dim, A, S, T = 5, 72, 12, 98, 20
    keys, grouping, model = _product_model(n, obs_dim, A, S)
    cfg = Namespace(distributed_training=False, episode_length=T, use_grad_clip=True, grad_clip_norm=10.0,
                    device=DEV, model_dir="/tmp/x", running_steps=100000, parallels=4, use_parameter_sharing=True,
                    use_rnn=True, use_actions_mask=False, learning_rate=7e-4, sync_frequency=1, double_q=True,
                    n_epochs=1, start_training=0, gamma=0.99, end_factor_lr_decay=0.5, qmix_rnn_detach_q_eval=False,
                    use_cuda_graph=False)
    lrn = QMIX_Learner(cfg, grouping, model, BaseCallback())
    prod, _ = _buffers(keys, obs_dim, A, S, 4, 16, 8, T)
    for ev in qmix_episode_stream(np.random.default_rng(3), keys, 4, T, obs_dim, A, S, 4):
        if ev[0] == 'store':
            prod.store(**ev[1])
        else:
            prod.finish_path(ev[1], **ev[2])
    seen = []
    inner = model.Qtarget_tot

    def record(q_taken, states):
        out = inner(q_taken, states)
        params = {k: v.clone() for k, v in model.target_Qtot.state_dict().items()}
        seen.append((q_taken.detach().clone(), states.detach().clone(), out.detach().clone(), params))
        return out

    model.Qtarget_tot = record
    np.random.seed(0)
    lrn.update(prod.sample())            # sync_frequency = 1: the target mixer now equals the trained eval mixer
    seen.clear()
    lrn.update(prod.sample())
    q_t, s_t, got, params = seen[0]
    tm = _mixer(S, n, False)
    tm.load_state_dict(params)           # the target mixer as that update saw it
    q = q_t.reshape(-1, n).cpu().numpy()
    st = s_t.reshape(-1, S).cpu().numpy()
    _check(tm, q, st, got.reshape(-1).cpu().numpy(), "learner Qtarget_tot, K9-TC")
    tm.use_tensor_core_forward = False
    try:
        with torch.no_grad():
            plain = tm(q_t, s_t).reshape(-1).cpu().numpy()
    finally:
        tm.use_tensor_core_forward = True
    _check(tm, q, st, plain, "learner Qtarget_tot, cuBLAS + K9")

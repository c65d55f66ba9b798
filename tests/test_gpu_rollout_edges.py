"""GPU: the rollout-side kernels (K2 xb_gae_scan, the GAE path of xb_gae_scan_vn, K10 xb_categorical_act, K11
xb_rms_update_normalize) called through the C-ABI against tests/rollout_refs.py, at their tile, tier and masking edges:
T at the lane (4) and tile (128) boundaries and up to 16 tiles, segment ends and terminals on those boundaries, the
float4 and the scalar load paths, every K10 template tier, masked logits and the uniforms 0 and 1 - 2^-24, and K11's
cancellation and count regimes.

Tolerances.  EPS = 2^-24.  K2's float32 GAE is held to rollout_refs.gae_bound (derivation in its docstring), its ret to
that plus EPS |ret|; its non-GAE adv (one float32 residual of three roundings) to 3 EPS (1 + 4 EPS) D_t.  The float64
scans (K2's returns, xb_gae_scan_vn) round once to float32: within one float32 ulp of the float64 reference plus the
same bound evaluated at float64's unit roundoff.  K10's logp, entropy and draws are held to
rollout_refs.categorical_bounds.  K11 follows the header's float32 operation order with correctly rounded operations,
so it is compared bit for bit."""
import numpy as np
import pytest
import torch

import rollout_refs as rr
from mappo_refs import denorm_f32, mean_std_f32

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = rr.EPS32
f32 = np.float32
GL = [(0.99, 0.95), (0.98, 0.95), (1.0, 1.0)]
T_SET = [1, 3, 4, 127, 128, 129, 255, 256, 257, 2048]
N_SET = [1, 3, 4, 5, 257]


def _lib():
    from xuance_b200 import _lib
    return _lib


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _within(got, want, tol, what):
    got = np.asarray(got.cpu().numpy() if torch.is_tensor(got) else got, np.float64)
    want, tol = np.broadcast_to(np.asarray(want, np.float64), got.shape), np.broadcast_to(tol, got.shape)
    err = np.abs(got - want)
    bad = ~(err <= tol)                       # NaN (an unwritten output) fails too
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, np.nan_to_num(err / np.maximum(tol, 1e-300), nan=np.inf), 0)), got.shape)
        raise AssertionError(f"{what}: {bad.sum()} of {bad.size} outside tolerance; at {i}: got {got[i]!r} want {want[i]!r} "
                             f"tol {tol[i]!r}")


def _bits(t):
    return t.cpu().numpy().view(np.uint32) if t.dtype == torch.float32 else t.cpu().numpy()


def _dev(x, offset):
    """x on the device; offset=1 places it one element past a 256-byte aligned allocation (no 16-byte alignment)."""
    flat = np.ascontiguousarray(x).reshape(-1)
    buf = torch.zeros(flat.size + offset, dtype=torch.from_numpy(flat[:0]).dtype, device=DEV)
    buf[offset:] = torch.from_numpy(flat).to(DEV)
    return buf[offset:].view(x.shape)


def _out(shape, offset, fill=float("nan")):
    buf = torch.full((int(np.prod(shape)) + offset,), fill, device=DEV)
    return buf[offset:].view(shape)


# ------------------------------------------------------------------------------------------------------ K2
def _run_gae(c, rows, gamma, lam, use_gae, offset):
    N, T = len(rows), c["rew"].shape[1]
    ins = [_dev(c[k][rows], offset) for k in ("rew", "val", "term", "seg_end", "boot")]
    cov = _t(c["covered"][rows])
    adv, ret = _out((N, T), offset), _out((N, T), offset)
    _lib().call("xb_gae_scan", *[_lib().ptr(x) for x in ins], _lib().ptr(cov), _lib().ptr(adv), _lib().ptr(ret), N, T,
                gamma, lam, int(use_gae))
    return adv, ret


@pytest.mark.parametrize("use_gae", [True, False])
@pytest.mark.parametrize("gamma,lam", GL)
@pytest.mark.parametrize("T", T_SET)
def test_gae_scan_edges(T, gamma, lam, use_gae):
    rng = np.random.default_rng(T * 10 + int(use_gae))
    for N in N_SET:
        c = rr.gae_case(rng, N, T)
        rows = np.arange(N)
        adv, ret = _run_gae(c, rows, gamma, lam, use_gae, 0)
        a64, r64 = rr.gae_scan(c["rew"], c["val"], c["term"], c["seg_end"], c["boot"], c["covered"], gamma, lam,
                               use_gae)
        live = np.arange(T)[None, :] < c["covered"][:, None]
        what = f"N={N} T={T} use_gae={use_gae}"
        an, rn = adv.cpu().numpy(), ret.cpu().numpy()
        # steps at or beyond covered are exactly +0
        assert np.all(_bits(adv)[~live] == 0) and np.all(_bits(ret)[~live] == 0), what
        coef = rr.gae_coef(c["term"], c["seg_end"], gamma, lam, use_gae)
        L = rr.scan_levels(T)
        if use_gae:
            b = rr.gae_bound(coef, rr.gae_mag(c["rew"], c["val"], c["seg_end"], c["boot"], gamma), L)
            _within(an, a64, np.where(live, b, 0), "adv " + what)
            _within(rn, r64, np.where(live, b * (1 + EPS) + EPS * np.abs(r64), 0), "ret " + what)
        else:
            mag = rr.gae_mag(c["rew"], c["val"], c["seg_end"], c["boot"], gamma)
            _within(an, a64, np.where(live, 3 * EPS * (1 + 4 * EPS) * mag, 0), "adv " + what)
            b64 = rr.gae_bound(coef, rr.gae_mag(c["rew"], c["val"], c["seg_end"], c["boot"], gamma, False), L,
                               rr.EPS64)
            _within(rn, r64, np.where(live, rr.ulp32(r64) + b64, 0), "ret " + what)
        # the scalar load path (operands one float past 16-byte alignment) gives the same bits as the float4 path
        adv_s, ret_s = _run_gae(c, rows, gamma, lam, use_gae, 1)
        assert np.array_equal(_bits(adv_s), _bits(adv)) and np.array_equal(_bits(ret_s), _bits(ret)), what
        # launch to launch, and a row alone vs. inside the batch
        adv2, ret2 = _run_gae(c, rows, gamma, lam, use_gae, 0)
        assert np.array_equal(_bits(adv2), _bits(adv)) and np.array_equal(_bits(ret2), _bits(ret)), what
        for n in {0, N // 2, N - 1}:
            adv1, ret1 = _run_gae(c, np.array([n]), gamma, lam, use_gae, n % 2)
            assert np.array_equal(_bits(adv1)[0], _bits(adv)[n]) and np.array_equal(_bits(ret1)[0], _bits(ret)[n])


# ------------------------------------------------------------------------------------------------------ K2 (ValueNorm)
SENTINEL = 12345.5


@pytest.mark.parametrize("value_norm", [False, True])
@pytest.mark.parametrize("T", T_SET)
def test_gae_scan_vn_edges(T, value_norm):
    rng = np.random.default_rng(T * 3 + int(value_norm))
    gamma, lam = 0.99, 0.95
    vn_state = (f32(0.3), f32(2.0), f32(0.9)) if value_norm else None
    vn = mean_std_f32(*vn_state) if value_norm else None
    for N in N_SET:
        c = rr.gae_case(rng, N, T)
        start = np.zeros(N, np.int32)
        if T > 1:
            start[1::2] = rng.integers(0, c["covered"][1::2])      # start > 0 (< covered) on every other row
        adv, ret = _out((N, T), 0, SENTINEL), _out((N, T), 0, SENTINEL)
        ins = [_t(c[k]) for k in ("rew", "val", "term", "seg_end", "boot")]
        st = [_t(np.array([x], f32)) for x in vn_state] if value_norm else [None] * 3
        d_start, d_cov = _t(start), _t(c["covered"])
        _lib().call("xb_gae_scan_vn", *[_lib().ptr(x) for x in ins], _lib().ptr(d_start), _lib().ptr(d_cov),
                    _lib().ptr(adv), _lib().ptr(ret), N, T, gamma, lam, 1, *[_lib().ptr(x) for x in st])
        v_dn, b_dn = denorm_f32(c["val"], vn), denorm_f32(c["boot"], vn)
        r64, coef, mag = rr.gae_vn(c["rew"], v_dn, c["term"], c["seg_end"], b_dn, gamma, lam)
        tt = np.arange(T)[None, :]
        win = (tt >= start[:, None]) & (tt < c["covered"][:, None])
        an, rn = adv.cpu().numpy(), ret.cpu().numpy()
        what = f"N={N} T={T} vn={value_norm}"
        assert np.all(an[~win] == SENTINEL) and np.all(rn[~win] == SENTINEL), what
        # one rounding of the float64 scan (its own error: gae_bound at float64's unit roundoff, plus the final addition)
        b64 = rr.gae_bound(coef, mag, rr.scan_levels(T), rr.EPS64) + rr.EPS64 * np.abs(r64)
        _within(rn, np.where(win, r64, SENTINEL), np.where(win, rr.ulp32(r64) + b64, 0), "ret " + what)
        assert np.array_equal(an[win], (rn - v_dn)[win]), what      # adv = f32(ret - V) exactly


# ------------------------------------------------------------------------------------------------------ K10
A_SET = [1, 2, 3, 4, 5, 8, 9, 18, 19, 32, 33, 63, 64]
N_ACT = [1, 127, 128, 129, 4097]


def _act(z, u=None, forced=None, outs=("f", "i", "lp", "ent")):
    N, A = z.shape
    o = {"f": _out((N,), 0), "i": torch.full((N,), -7, dtype=torch.int32, device=DEV), "lp": _out((N,), 0),
         "ent": _out((N,), 0)}
    p = {k: (v if k in outs else None) for k, v in o.items()}
    d_z, d_u, d_f = _t(z), (None if u is None else _t(u)), (None if forced is None else _t(forced))
    _lib().call("xb_categorical_act", _lib().ptr(d_z), _lib().ptr(d_u), _lib().ptr(d_f), N, A,
                *[_lib().ptr(p[k]) for k in ("f", "i", "lp", "ent")])
    return {k: p[k] for k in outs}


def _act_logits(rng, N, A):
    """Spread logits; every 9th row shifted by +1e4, every 9th (offset 4) by -1e4; every 5th row with its maximum tied
    at the first and the last index."""
    z = (rng.normal(size=(N, A)) * 3).astype(f32)
    if A > 1:
        r = np.arange(2, N, 5)
        z[r, 0] = z[r, A - 1] = z[r].max(axis=1) + f32(0.5)
    z[0::9] += f32(1e4)
    z[4::9] -= f32(1e4)
    return z


@pytest.mark.parametrize("A", A_SET)
def test_categorical_act_edges(A):
    rng = np.random.default_rng(A)
    for N in N_ACT:
        z = _act_logits(rng, N, A)
        u = rng.random(N).astype(f32)
        u[0::4], u[1::4] = 0.0, 1 - 2.0 ** -24
        lp64, p64, ent64, _ = rr.categorical(z)
        E, ent_b, delta = rr.categorical_bounds(z)
        rows = np.arange(N)
        what = f"N={N} A={A}"
        o = _act(z, u)
        a = o["i"].cpu().numpy().astype(np.int64)
        assert np.array_equal(o["f"].cpu().numpy(), a.astype(f32)), what
        assert np.all((a >= 0) & (a < A)) and np.all(p64[rows, a] > 0), what
        assert np.all(rr.draw_allowed(p64, u, delta, a)), what
        sure = np.abs(np.cumsum(p64, axis=1) - u[:, None].astype(np.float64)).min(axis=1) > delta
        assert np.array_equal(a[sure], rr.draw(p64, u)[sure]), what
        _within(o["lp"], lp64[rows, a], E[rows, a], "logp " + what)
        _within(o["ent"], ent64, ent_b, "entropy " + what)
        # each output alone gives the same bits as all four together
        for k in ("f", "i", "lp", "ent"):
            assert np.array_equal(_bits(_act(z, u, outs=(k,))[k]), _bits(o[k])), what + " " + k
        # argmax: the first maximal index; exact where the top two probabilities are farther apart than their error
        d = _act(z)
        a_d = d["i"].cpu().numpy().astype(np.int64)
        perr = p64 * (E + 4 * EPS)
        top = np.sort(p64, axis=1)
        gap_ok = (top[:, -1] - (top[:, -2] if A > 1 else 0)) > 2 * perr.max(axis=1)
        first = rr.argmax_first(z)
        tie = np.zeros(N, bool)
        if A > 1:
            tie[np.arange(2, N, 5)] = True
            assert np.all(a_d[tie] == 0), what
        assert np.array_equal(a_d[gap_ok], first[gap_ok]), what
        assert np.all(p64[rows, a_d] >= p64[rows, first] - 2 * perr.max(axis=1)), what
        _within(d["lp"], lp64[rows, a_d], E[rows, a_d], "argmax logp " + what)
        # forced actions: logp of the given action
        forced = rng.integers(0, A, N)
        fo = _act(z, forced=forced.astype(f32), outs=("lp", "ent"))
        _within(fo["lp"], lp64[rows, forced], E[rows, forced], "forced logp " + what)
        assert np.array_equal(_bits(fo["ent"]), _bits(o["ent"])), what


@pytest.mark.parametrize("A", [9, 12, 19])
def test_categorical_act_never_draws_a_masked_action(A):
    """The SMAC layout: the first action and the last three at -1e10.  With u = 1 - 2^-24 no prefix of the float32 CDF
    need pass u, and the draw must then be the last AVAILABLE action (given probability >= 1e-3, so that it is also the
    float64 draw); with u = 0 it must be the first available action."""
    rng = np.random.default_rng(A)
    N = 4096
    z = (rng.normal(size=(N, A)) * 2).astype(f32)
    avail = np.arange(1, A - 3)
    z[:, A - 4] = np.maximum(z[:, A - 4], z[:, avail].max(axis=1) - 4)      # p >= e^-4 / (A - 4) >= 1e-3
    z[:, [0, A - 3, A - 2, A - 1]] = -1e10
    u = np.full(N, 1 - 2.0 ** -24, f32)
    u[::8] = 0.0
    o = _act(z, u)
    a = o["i"].cpu().numpy()
    p64 = rr.categorical(z)[1]
    assert p64[:, A - 4].min() >= 1e-3
    want = np.where(u == 0, 1, A - 4)
    bad = a != want
    assert not bad.any(), f"{bad.sum()} of {N} rows drew action(s) {np.unique(a[bad])}"
    E = rr.categorical_bounds(z)[0]
    _within(o["lp"], rr.categorical(z)[0][np.arange(N), a], E[np.arange(N), a], "logp")


def test_categorical_act_minus_inf_logits():
    """-inf logits (masked_fill): the entropy is torch's finite one, the draw never picks a -inf action."""
    rng = np.random.default_rng(3)
    N, A = 1000, 7
    z = (rng.normal(size=(N, A)) * 2).astype(f32)
    z[:, 0] = -np.inf
    z[1::2, A - 1] = -np.inf
    z[2::3, 3] = -np.inf
    u = rng.random(N).astype(f32)
    u[::3] = 1 - 2.0 ** -24
    o = _act(z, u)
    lp64, p64, ent64, _ = rr.categorical(z)
    E, ent_b, delta = rr.categorical_bounds(z)
    want = torch.distributions.Categorical(logits=torch.from_numpy(z).double()).entropy().numpy()
    np.testing.assert_allclose(ent64, want, rtol=1e-12, atol=1e-12)
    _within(o["ent"], want, ent_b, "entropy")
    a = o["i"].cpu().numpy().astype(np.int64)
    assert np.all(np.isfinite(z[np.arange(N), a])) and np.all(rr.draw_allowed(p64, u, delta, a))
    _within(o["lp"], lp64[np.arange(N), a], E[np.arange(N), a], "logp")


def test_categorical_act_status_codes():
    lib = _lib().load()
    z = torch.zeros((4, 65), device=DEV)
    o = torch.zeros(4, device=DEV)
    assert lib.xb_categorical_act(z.data_ptr(), None, None, 4, 65, o.data_ptr(), None, None, None, None) == -3
    assert lib.xb_categorical_act(z.data_ptr(), None, None, 0, 4, o.data_ptr(), None, None, None, None) == -1


# ------------------------------------------------------------------------------------------------------ K11
def _rms(x, mean, var, count, update, out, clip=5.0):
    N, D = x.shape
    m, v = _t(mean), _t(var)
    y = _out((N, D), 0) if out else None
    d_x = _t(x)
    _lib().call("xb_rms_update_normalize", _lib().ptr(d_x), N, D, _lib().ptr(m), _lib().ptr(v), count, int(update),
                _lib().ptr(y), clip, 1e-8)
    return m.cpu().numpy(), v.cpu().numpy(), (y.cpu().numpy() if out else None)


@pytest.mark.parametrize("D", [1, 127, 128, 129, 1000])
@pytest.mark.parametrize("N", [1, 2, 256])
def test_rms_update_normalize_bit_exact(N, D):
    """Against the float32 loop in the header's order: constant columns, a 1e4 offset with 1e-2 noise, counts of 1e-4,
    2^24 + 3 and 1e9, clip saturation (a clip range at the median |output|), and update-only / output-only calls."""
    rng = np.random.default_rng(N * 7 + D)
    mean = (rng.normal(size=D) * 0.1).astype(f32)
    var = (rng.random(D) + 0.5).astype(f32)
    for it, count in enumerate([1e-4, 2.0 ** 24 + 3, 1e9]):
        x = (rng.normal(size=(N, D)) * (1e-2 if it == 1 else 3.0) + (1e4 if it == 1 else 0.0)).astype(f32)
        x[:, 1::7] = f32(0.3) if it != 1 else f32(1e4)                 # constant columns
        m_ref, v_ref = rr.rms_update_f32(x, mean, var, count)
        clip = float(np.median(np.abs(rr.rms_normalize_f32(x, m_ref, v_ref, 1e30)))) if it == 2 else 5.0
        y_ref = rr.rms_normalize_f32(x, m_ref, v_ref, clip)
        m, v, y = _rms(x, mean, var, count, True, True, clip)
        assert np.array_equal(m.view(np.uint32), m_ref.view(np.uint32)) and np.array_equal(v.view(np.uint32),
                                                                                            v_ref.view(np.uint32))
        assert np.array_equal(y.view(np.uint32), y_ref.view(np.uint32))
        if it == 2 and N * D > 1:
            assert (np.abs(y) == f32(clip)).any()
        m_u, v_u, _ = _rms(x, mean, var, count, True, False)
        assert np.array_equal(m_u, m_ref) and np.array_equal(v_u, v_ref)
        m_o, v_o, y_o = _rms(x, m_ref, v_ref, count, False, True, clip)
        assert np.array_equal(m_o, m_ref) and np.array_equal(v_o, v_ref)
        assert np.array_equal(y_o.view(np.uint32), y_ref.view(np.uint32))
        mean, var = m_ref, v_ref

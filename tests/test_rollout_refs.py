"""CPU: pins tests/rollout_refs.py - the float64 GAE against the oracle's finish_path, the categorical reference against
torch.distributions.Categorical, the K11 float32 loop against the oracle's RunningMeanStd - and shows that the derived
bounds hold for float32 models of the kernels' evaluation orders and fail for a scan with its tile carry dropped or
shifted, so that a wrong reference or a slack bound cannot make tests/test_gpu_rollout_edges.py pass."""
import numpy as np
import pytest
import torch

import rollout_refs as rr
from oracle.onpolicy import gae_segment
from oracle.rollout import RunningMeanStdOracle, process_observation

f32 = np.float32
U = rr.EPS32
GL = [(0.99, 0.95), (0.98, 0.95), (1.0, 1.0)]


def _segments(se_row, cov):
    """(first, last) steps of the finished paths of one row."""
    out, s = [], 0
    for t in range(cov):
        if se_row[t]:
            out.append((s, t))
            s = t + 1
    return out


def _oracle_rows(c, gamma, lam):
    adv, ret = np.zeros(c["rew"].shape, f32), np.zeros(c["rew"].shape, f32)
    for n in range(c["rew"].shape[0]):
        for s, e in _segments(c["seg_end"][n], c["covered"][n]):
            a, r = gae_segment(c["rew"][n, s:e + 1], c["val"][n, s:e + 1], c["term"][n, s:e + 1], c["boot"][n, e],
                               gamma, lam)
            adv[n, s:e + 1], ret[n, s:e + 1] = a, r
    return adv, ret


@pytest.mark.parametrize("T", [1, 37, 300])
def test_gae_equals_oracle_exactly_on_dyadic_paths(T):
    """gamma = lam = 1 and small integers: every float32 operation of the oracle is exact, so the float64 reference must
    equal it bit for bit - segment ends, terminals, bootstraps and covered all placed as the oracle places them."""
    rng = np.random.default_rng(T)
    c = rr.gae_case(rng, 10, T)
    for k in ("rew", "val", "boot"):
        c[k] = rng.integers(-8, 9, c[k].shape).astype(f32)
    adv, ret = rr.gae_scan(c["rew"], c["val"], c["term"], c["seg_end"], c["boot"], c["covered"], 1.0, 1.0, True)
    a_o, r_o = _oracle_rows(c, 1.0, 1.0)
    assert np.array_equal(adv, a_o.astype(np.float64)) and np.array_equal(ret, r_o.astype(np.float64))


@pytest.mark.parametrize("gamma,lam", GL)
@pytest.mark.parametrize("T", [129, 1000])
def test_gae_equals_oracle_within_sequential_bound(T, gamma, lam):
    """On random paths the oracle's sequential float32 loop is within gae_bound with L = 2 of the float64 reference
    (derivation in rollout_refs.gae_bound), and the bound is not vacuous: for gamma*lam < 1 it is below 1e-3 of the
    values' scale (at gamma*lam = 1 the worst case grows as T^2 along a path)."""
    rng = np.random.default_rng(T + int(gamma * 100))
    c = rr.gae_case(rng, 10, T)
    adv, ret = rr.gae_scan(c["rew"], c["val"], c["term"], c["seg_end"], c["boot"], c["covered"], gamma, lam, True)
    a_o, _ = _oracle_rows(c, gamma, lam)
    b = rr.gae_bound(rr.gae_coef(c["term"], c["seg_end"], gamma, lam),
                     rr.gae_mag(c["rew"], c["val"], c["seg_end"], c["boot"], gamma), 2)
    assert np.all(np.abs(a_o - adv) <= b)
    assert gamma * lam == 1 or b.max() < 1e-3 * np.abs(adv).max()


def _delta32(c, gamma):
    """K2's float32 delta_t = r_t + (1-d_t)*gamma*V'_t - V_t (without contraction)."""
    se = c["seg_end"] != 0
    vn = np.where(se, c["boot"], np.concatenate([c["val"][:, 1:], np.zeros((c["val"].shape[0], 1), f32)], axis=1))
    nd = f32(1) - c["term"]
    return (c["rew"] + (nd * f32(gamma)) * vn) - c["val"]


def _warp_scan_f32(b, a, drop_carry=False):
    """Float32 model of K2's evaluation order (csrc/rollout.cu gae_scan_kernel, one multiplication and one addition per
    composition where the device may fuse them): 4 serial steps per lane, a 5-level shuffle scan from the high lanes
    down, the exclusive prefix applied to the carry, each lane's local maps applied, lane 0's first value carried into
    the previous 128-step tile."""
    N, T = b.shape
    nt = -(-T // rr.TILE)
    bp, ap = np.zeros((N, nt * rr.TILE), f32), np.zeros((N, nt * rr.TILE), f32)
    bp[:, :T], ap[:, :T] = b, a
    out = np.zeros_like(bp)
    carry = np.zeros(N, f32)
    for tile in range(nt - 1, -1, -1):
        sl = slice(tile * rr.TILE, (tile + 1) * rr.TILE)
        fb, fa = bp[:, sl].reshape(N, 32, 4), ap[:, sl].reshape(N, 32, 4)
        la, lb = np.zeros_like(fa), np.zeros_like(fb)
        acc_a, acc_b = np.ones((N, 32), f32), np.zeros((N, 32), f32)
        for j in range(3, -1, -1):
            acc_a, acc_b = fa[:, :, j] * acc_a, fa[:, :, j] * acc_b + fb[:, :, j]
            la[:, :, j], lb[:, :, j] = acc_a, acc_b
        inc_a, inc_b = acc_a, acc_b
        for o in (1, 2, 4, 8, 16):
            oa, ob = np.ones_like(inc_a), np.zeros_like(inc_b)
            oa[:, :32 - o], ob[:, :32 - o] = inc_a[:, o:], inc_b[:, o:]
            inc_a, inc_b = inc_a * oa, inc_a * ob + inc_b
        ex_a, ex_b = np.ones_like(inc_a), np.zeros_like(inc_b)
        ex_a[:, :31], ex_b[:, :31] = inc_a[:, 1:], inc_b[:, 1:]
        x_in = ex_a * (f32(0) if drop_carry else carry)[..., None] + ex_b
        y = la * x_in[:, :, None] + lb
        out[:, sl] = y.reshape(N, rr.TILE)
        carry = y[:, 0, 0]
    return out[:, :T]


@pytest.mark.parametrize("gamma,lam", GL)
@pytest.mark.parametrize("T", [127, 256, 2048])
def test_gae_bound_holds_for_the_scan_order_and_discriminates(T, gamma, lam):
    """The derived bound (L = scan_levels(T)) holds for a float32 model of the warp scan, and is violated at these shapes
    by a scan whose tile carry is dropped or taken one step late (A_{t+2} instead of A_{t+1} at a tile edge)."""
    rng = np.random.default_rng(T)
    c = rr.gae_case(rng, 10, T, short=False)
    adv, _ = rr.gae_scan(c["rew"], c["val"], c["term"], c["seg_end"], c["boot"], None, gamma, lam, True)
    coef = rr.gae_coef(c["term"], c["seg_end"], gamma, lam)
    b = rr.gae_bound(coef, rr.gae_mag(c["rew"], c["val"], c["seg_end"], c["boot"], gamma), rr.scan_levels(T))
    a32 = np.where(c["seg_end"] != 0, f32(0), (f32(1) - c["term"]) * rr.gl32(gamma, lam))
    model = _warp_scan_f32(_delta32(c, gamma), a32)
    assert np.all(np.abs(model - adv) <= b)
    if T <= rr.TILE:
        return
    edge = (np.arange(T) % rr.TILE) == rr.TILE - 1
    dropped = rr.gae_scan(c["rew"], c["val"], c["term"], c["seg_end"], c["boot"], None, gamma, lam, True,
                          coef=np.where(edge, 0.0, coef))[0]
    assert (np.abs(dropped - adv) > b).any()
    assert (np.abs(_warp_scan_f32(_delta32(c, gamma), a32, drop_carry=True) - adv) > b).any()
    late = adv.copy()       # A_t = delta_t + c_t * A_{t+2} at t = 127 mod 128
    t = np.nonzero(edge)[0]
    t = t[t + 2 < T]
    late[:, t] = adv[:, t] - coef[:, t] * adv[:, t + 1] + coef[:, t] * adv[:, t + 2]
    assert (np.abs(late - adv) > b).any()


def test_gae_returns_path_matches_discounted_returns():
    """use_gae=0: ret equals the oracle's float64 lfilter recurrence per segment, adv its one-step residual."""
    from oracle.onpolicy import discounted_returns
    rng = np.random.default_rng(5)
    c = rr.gae_case(rng, 10, 300)
    gamma = 0.99
    adv, ret = rr.gae_scan(c["rew"], c["val"], c["term"], c["seg_end"], c["boot"], c["covered"], gamma, 0.95, False)
    g = float(f32(gamma))
    for n in range(10):
        for s, e in _segments(c["seg_end"][n], c["covered"][n]):
            rw = np.append(c["rew"][n, s:e + 1].astype(np.float64), c["boot"][n, e])
            vs = np.append(c["val"][n, s:e + 1].astype(np.float64), c["boot"][n, e])
            np.testing.assert_allclose(ret[n, s:e + 1], discounted_returns(rw, g)[:-1], rtol=1e-14, atol=1e-14)
            np.testing.assert_allclose(adv[n, s:e + 1], rw[:-1] + g * vs[1:] - vs[:-1], rtol=1e-15, atol=1e-15)
        assert not ret[n, c["covered"][n]:].any() and not adv[n, c["covered"][n]:].any()


# ------------------------------------------------------------------------------------------------------ K10
def _logits(rng, N, A):
    """Spread logits with exact ties, -1e10 and -inf masks (never the whole row) and rows shifted by +-1e4."""
    z = (rng.normal(size=(N, A)) * 3).astype(f32)
    if A > 1:
        z[0::7, 1] = z[0::7, 0] = np.maximum(z[0::7, 0], z[0::7].max(axis=1))     # tie at the maximum
        z[1::7, A - 1] = -1e10
        z[2::7, 0] = -np.inf
        z[3::7, A // 2:] = -1e10
    z[4::7] += f32(1e4)
    z[5::7] -= f32(1e4)
    return z


@pytest.mark.parametrize("A", [1, 2, 5, 12, 64])
def test_categorical_equals_torch(A):
    rng = np.random.default_rng(A)
    z = _logits(rng, 700, A)
    lp, p, ent, _ = rr.categorical(z)
    d = torch.distributions.Categorical(logits=torch.from_numpy(z).double())
    for i in range(A):
        want = d.log_prob(torch.full((700,), i)).numpy()
        fin = np.isfinite(want)
        assert np.array_equal(fin, np.isfinite(lp[:, i]))
        np.testing.assert_allclose(lp[fin, i], want[fin], rtol=1e-13, atol=1e-11)
    assert np.all(np.isfinite(ent))
    np.testing.assert_allclose(ent, d.entropy().numpy(), rtol=1e-12, atol=1e-12)
    assert np.array_equal(rr.argmax_first(z), d.probs.argmax(dim=1).numpy())
    np.testing.assert_allclose(p, d.probs.numpy(), rtol=1e-12, atol=1e-300)


def test_categorical_draw_frequencies_and_fallback():
    """Empirical frequencies of the inverse-CDF draw follow torch's probabilities (5 sigma), masked categories are never
    drawn, and a u the CDF does not pass falls back to the last index with positive probability."""
    z = np.array([[-1e10, 0.5, -1.0, 2.0, 0.0, -np.inf, -1e10]], f32)
    n = 400000
    u = np.random.default_rng(0).random(n)
    a = rr.draw(np.repeat(rr.categorical(z)[1], n, axis=0), u)
    p = torch.distributions.Categorical(logits=torch.from_numpy(z).double()).probs.numpy()[0]
    freq = np.bincount(a, minlength=7) / n
    assert np.all(np.abs(freq - p) <= 5 * np.sqrt(p * (1 - p) / n))
    assert freq[0] == freq[5] == freq[6] == 0
    p1 = rr.categorical(z)[1]
    assert rr.draw(p1, np.array([1.0]))[0] == 4 and rr.draw(p1, np.array([0.0]))[0] == 1


def _act_f32(z, u, last_positive):
    """Float32 model of K10's loop (csrc/act.cu): sequential sums, a product and a sum per entropy term; the
    fall-through takes the last index with p > 0 (last_positive) or the last index (the rule before the fix)."""
    z = np.asarray(z, f32)
    N, A = z.shape
    m = z.max(axis=1)
    se = np.zeros(N, f32)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(A):
            se = se + np.exp(z[:, i] - m)
        lse = m + np.log(se)
        ent, cdf = np.zeros(N, f32), np.zeros(N, f32)
        a, lp_all = np.full(N, -1), np.zeros((N, A), f32)
        last = np.full(N, A - 1)
        for i in range(A):
            lp = z[:, i] - lse
            p = np.exp(lp)
            lp_all[:, i] = lp
            ent = np.where(p > 0, ent - p * lp, ent)
            cdf = cdf + p
            a = np.where((a < 0) & (u < cdf), i, a)
            if last_positive:
                last = np.where(p > 0, i, last)
    a = np.where(a < 0, last, a)
    return a, lp_all[np.arange(N), a], ent


@pytest.mark.parametrize("A", [1, 3, 12, 33, 64])
def test_categorical_bounds_hold_for_float32_model(A):
    """logp, entropy and the draw of a float32 model of K10 (NumPy's exp / log, within CUDA's documented 2 / 1 ulp) stay
    within categorical_bounds, including u = 0, u = 1 - 2^-24, masks and +-1e4 shifts."""
    rng = np.random.default_rng(100 + A)
    z = _logits(rng, 2000, A)
    u = rng.random(2000).astype(f32)
    u[::5], u[1::5] = 0.0, 1 - 2.0 ** -24
    lp, p, ent, _ = rr.categorical(z)
    E, ent_b, delta = rr.categorical_bounds(z)
    a, lp_a, ent_a = _act_f32(z, u, True)
    rows = np.arange(2000)
    assert np.all(np.abs(lp_a - lp[rows, a]) <= E[rows, a])
    assert np.all(np.abs(ent_a - ent) <= ent_b)
    assert np.all(rr.draw_allowed(p, u, delta, a))
    sure = np.abs(np.cumsum(p, axis=1) - u[:, None].astype(np.float64)).min(axis=1) > delta
    assert sure.mean() > 0.5 and np.array_equal(a[sure], rr.draw(p, u)[sure])


def test_draw_allowed_rejects_the_masked_fall_through():
    """With the last three of 12 actions masked and u = 1 - 2^-24, the old rule (fall through to A - 1) draws a
    masked action whenever the float32 total mass rounds below 1; draw_allowed flags each such row."""
    rng = np.random.default_rng(7)
    z = (rng.normal(size=(4096, 12)) * 2).astype(f32)
    z[:, [0, 9, 10, 11]] = -1e10
    u = np.full(4096, 1 - 2.0 ** -24, f32)
    p, delta = rr.categorical(z)[1], rr.categorical_bounds(z)[2]
    old = _act_f32(z, u, False)[0]
    assert (old == 11).sum() > 100
    assert not rr.draw_allowed(p, u, delta, old)[old == 11].any()
    assert np.all(rr.draw_allowed(p, u, delta, _act_f32(z, u, True)[0]))


# ------------------------------------------------------------------------------------------------------ K11
@pytest.mark.parametrize("D", [2, 3, 127, 128, 129, 1000])
@pytest.mark.parametrize("N", [1, 2, 7, 256])
def test_rms_loop_equals_oracle(N, D):
    """The row-after-row float32 loop equals RunningMeanStdOracle (NumPy's axis-0 mean / std) bit for bit, update and
    normalised output, across counts of 1e-4, 2^24 + 3 and 1e9, a 1e4 offset with 1e-2 noise and constant columns."""
    rng = np.random.default_rng(N * 1000 + D)
    orc = RunningMeanStdOracle((D,))
    mean, var = orc.mean.copy(), orc.var.copy()
    for it, count in enumerate([1e-4, 2.0 ** 24 + 3, 1e9, 17.0]):
        x = (rng.normal(size=(N, D)) * (1e-2 if it == 1 else 3.0) + (1e4 if it == 1 else 0.0)).astype(f32)
        x[:, 0] = f32(0.3)
        orc.count = count
        orc.update(x)
        mean, var = rr.rms_update_f32(x, mean, var, count)
        assert np.array_equal(mean, orc.mean) and np.array_equal(var, orc.var)
        assert np.array_equal(rr.rms_normalize_f32(x, mean, var, 5.0), process_observation(x, orc, 5))


def test_rms_single_column_below_eight_rows_equals_oracle():
    """D = 1: NumPy reduces a single column as one contiguous run, row after row only below 8 rows (from 8 rows on it
    sums pairwise with 8 accumulators, an order K11 does not follow)."""
    rng = np.random.default_rng(1)
    for N in range(1, 8):
        orc = RunningMeanStdOracle((1,))
        x = (rng.normal(size=(N, 1)) * 3 + 1).astype(f32)
        orc.update(x)
        mean, var = rr.rms_update_f32(x, np.zeros(1, f32), np.ones(1, f32), 1e-4)
        assert np.array_equal(mean, orc.mean) and np.array_equal(var, orc.var)

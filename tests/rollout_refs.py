"""Float64 restatements of the rollout-side kernels' contracts as include/xb200.h states them (K2 xb_gae_scan, the GAE
path of xb_gae_scan_vn, K10 xb_categorical_act), the float32 restatement of K11 xb_rms_update_normalize in the header's
operation order, and the error bounds the GPU tests hold the float32 kernels to.  Inputs are NumPy arrays (float32 as
the kernels take them); every function returns NumPy arrays.  tests/test_rollout_refs.py pins these against the oracle
and torch.distributions on the CPU, and tests/test_gpu_rollout_edges.py compares the kernels with them.

Contracts restated here:
  * K2, use_gae=1:  delta_t = r_t + (1-d_t)*gamma*V'_t - V_t,  A_t = delta_t + c_t*A_{t+1},  c_t = (1-d_t)*gl,
                    ret_t = A_t + V_t;  V'_t = bootstrap_t where seg_end_t (and c_t = 0 there), else V_{t+1}
                    (0 beyond T).  gamma is the float32 the kernel receives and gl = f32(f32(gamma)*f32(lam)) its
                    float32 product, so the comparison measures arithmetic only.
  * K2, use_gae=0:  ret_t = r_t + gamma*(bootstrap_t if seg_end_t else ret_{t+1}) (terminals do not enter, as in
                    scipy.lfilter's discounted returns), adv_t = r_t + gamma*V'_t - V_t.
  * both:           steps at or beyond covered[n] are 0.
  * K10:            torch.distributions.Categorical(logits=z): lp = z - logsumexp(z), p = exp(lp),
                    entropy = -sum_{p_i > 0} p_i lp_i, argmax = first maximal index, inverse-CDF draw on a supplied u:
                    the first i with u < p_0 + .. + p_i; if no prefix passes u, the last index with p > 0.  A category
                    with p = 0 is never drawn.
  * K11:            RunningMeanStd.update + _process_observation in float32, the sums taken row after row.
"""
import numpy as np

f32, f64 = np.float32, np.float64
EPS32 = 2.0 ** -24          # unit roundoff of float32
EPS64 = 2.0 ** -53          # unit roundoff of float64
TILE = 128                  # K2's steps per warp tile (32 lanes x 4 steps)
TINY32 = 2.0 ** -149        # float32's smallest subnormal: expf's absolute error floor in the underflow range


def _d(x):
    return np.asarray(x, dtype=f64)


def gl32(gamma, lam):
    """The float32 product gamma*lam K2 forms from its float32 arguments."""
    return f32(f32(gamma) * f32(lam))


# ------------------------------------------------------------------------------------------------------ K2
def _backward(b, c):
    """x_t = b_t + c_t x_{t+1} from the back of each row, x_T = 0, in float64."""
    N, T = b.shape
    out = np.zeros((N, T))
    carry = np.zeros(N)
    for t in range(T - 1, -1, -1):
        carry = b[:, t] + c[:, t] * carry
        out[:, t] = carry
    return out


def gae_scan(rew, val, term, seg_end, boot, covered, gamma, lam, use_gae, coef=None):
    """xb_gae_scan in float64 as a plain per-segment backward loop over [N, T] inputs.  Returns (adv, ret) float64.
    gamma / lam are the float32 values the kernel receives (the GAE coefficient is gl32).  ``coef`` overrides the
    per-step coefficient c_t (use_gae only; tests build deliberately wrong scans with it)."""
    r, v, d, b = _d(rew), _d(val), _d(term), _d(boot)
    se = np.asarray(seg_end) != 0
    N, T = r.shape
    g = f64(f32(gamma))
    vnext = np.concatenate([v[:, 1:], np.zeros((N, 1))], axis=1)
    vnext = np.where(se, b, vnext)
    if use_gae:
        c = np.where(se, 0.0, (1.0 - d) * f64(gl32(gamma, lam))) if coef is None else _d(coef)
        delta = r + (1.0 - d) * g * vnext - v
    else:
        c = np.where(se, 0.0, g)
        delta = np.where(se, r + g * b, r)
    acc = _backward(delta, c)
    if use_gae:
        adv, ret = acc, acc + v
    else:
        adv, ret = r + g * vnext - v, acc
    cov = np.full(N, T) if covered is None else np.asarray(covered)
    live = np.arange(T)[None, :] < cov[:, None]
    return np.where(live, adv, 0.0), np.where(live, ret, 0.0)


def gae_vn(rew, val_dn, term, seg_end, boot_dn, gamma, lam):
    """The GAE path of xb_gae_scan_vn in float64 on the float32-denormalised values and bootstraps (val_dn, boot_dn):
    delta_t = r_t + (1-d_t)*gamma*V'_t - V_t, A_t = delta_t + (1-d_t)*gamma*lam*A_{t+1} with the float64 gamma and
    lam the kernel receives (0 at a segment end).  Returns (ret float64, coef, mag) for the whole row; the kernel
    writes f32(ret) and f32(ret) - V in float32 on [start, covered) only."""
    r, v, d, b = _d(rew), _d(val_dn), _d(term), _d(boot_dn)
    se = np.asarray(seg_end) != 0
    N = r.shape[0]
    vnext = np.where(se, b, np.concatenate([v[:, 1:], np.zeros((N, 1))], axis=1))
    c = np.where(se, 0.0, (1.0 - d) * gamma * lam)
    ret = _backward(r + (1.0 - d) * gamma * vnext - v, c) + v
    return ret, c, np.abs(r) + gamma * np.abs(vnext) + np.abs(v)


EDGES = (3, 4, 7, 8, 31, 32, 63, 64, 126, 127, 128, 129, 130, 131, 255, 256, 257, 1023, 1024, 2046)


def gae_case(rng, N, T, short=True):
    """[N, T] rollout fields for K2, one placement of segment ends and terminals per row (row n uses kind (n+1) % 5):
    0 sparse random; 1 at lane (t = 3 mod 4 / 0 mod 4) and tile (t = 127 / 128 ...) edges, terminals on the
    neighbouring edges; 2 a run of consecutive segment ends overlapping a run of consecutive terminals; 3 a segment
    end at every step; 4 one path over the whole row (the longest gamma*lam chain).  Every row ends a segment at
    covered - 1, as the buffer's finished paths do; with ``short`` every seventh row stops at covered < T and holds
    garbage beyond it.  Returns dict(rew, val, term, seg_end, boot, covered)."""
    rew = rng.normal(size=(N, T)).astype(f32)
    val = (rng.normal(size=(N, T)) * 3).astype(f32)
    boot = rng.normal(size=(N, T)).astype(f32)
    se = np.zeros((N, T), np.uint8)
    term = np.zeros((N, T), f32)
    edges = [t for t in EDGES if t < T]
    for n in range(N):
        kind = (n + 1) % 5
        if kind == 0:
            se[n] = rng.random(T) < 0.03
            term[n] = rng.random(T) < 0.03
        elif kind == 1:
            se[n, edges[0::2]] = 1
            term[n, edges[1::2]] = 1
        elif kind == 2:
            s = int(rng.integers(0, max(T - 8, 1)))
            se[n, s:s + 6] = 1
            term[n, s + 2:s + 9] = 1
        elif kind == 3:
            se[n] = 1
            term[n, ::3] = 1
    covered = np.full(N, T, np.int32)
    if short and T > 1:
        for n in range(6, N, 7):
            covered[n] = int(rng.integers(1, T))
    se[np.arange(N), covered - 1] = 1
    return dict(rew=rew, val=val, term=term, seg_end=se, boot=boot, covered=covered)


def gae_coef(term, seg_end, gamma, lam, use_gae=True):
    """The scan coefficients c_t of gae_scan: (1-d_t)*gl for GAE, gamma for the returns, 0 at a segment end."""
    se = np.asarray(seg_end) != 0
    if use_gae:
        return np.where(se, 0.0, (1.0 - _d(term)) * f64(gl32(gamma, lam)))
    return np.where(se, 0.0, f64(f32(gamma)))


def scan_levels(T):
    """L of gae_bound for K2's warp scan over T steps (see gae_bound): 4 + 5 + 1 + 1 + one per 128-step tile."""
    return 4 + 5 + 1 + 1 + -(-T // TILE)


def gae_bound(coef, mag, L, u=EPS32):
    """Per-element bound on |scan - exact| for the linear recurrence x_t = b_t + c_t x_{t+1} evaluated in precision u:
        bound(t) = 2u * sum_k (k + L) * |P_k| * D_{t+k},   P_k = c_t * c_{t+1} * ... * c_{t+k-1}  (P_0 = 1)
    with D_j = mag[j] a bound on |b_j| that also bounds b_j's own rounding error in units of 3u (for the GAE delta
    D_j = |r_j| + gamma*|V'_j| + |V_j|: three roundings, each at most u times a partial sum no larger than D_j).

    Derivation for K2 (csrc/rollout.cu).  Each lane composes its 4 steps serially, a 5-level shuffle scan composes the
    lanes, the exclusive prefix is applied to the carry entering the tile (x_in = E.a*carry + E.b), the lane applies
    its local map (y = loc.a*x_in + loc.b), and the tile's first y is the next tile's carry.  Follow one term
    P_k*b_{t+k} into x_t.  Every multiplication on its path multiplies by a composed coefficient that is a rounded
    product of a contiguous group of the c_j; a group of g coefficients costs g-1 roundings to form plus one to apply,
    and the groups partition the k coefficients, so the multiplications cost at most k roundings.  The additions: at
    most 3 inside the lane (the first composition is with the identity, exact), 5 in the shuffle levels, one for x_in,
    one for y, and two (x_in and y) for each further tile the term crosses: 10 + 2*(n_tiles - 1).  With b's own 3
    roundings the term carries relative error at most (k + 11 + 2*n_tiles) u, to first order, relative to
    |P_k| D_{t+k}.  L = 4 + 5 + 1 + 1 + n_tiles (scan_levels) gives 2(k + L) - (k + 11 + 2 n_tiles) = k + 11 > 0: the
    factor 2 (one multiplication and one addition per level) leaves at least 11u per term for the second-order terms,
    which are below (k + L)^2 u^2 and so below 1e-3 u at T <= 2048.  An FMA rounds once where the count charges two.

    The same bound with L = 2 holds for the sequential float32 loop of oracle.onpolicy.gae_segment: per step one
    multiplication and one addition, so (2k + 3) u for the term, and 2(k + 2) > 2k + 3.
    Evaluated in O(T) with S0_t = sum_k |P_k| D_{t+k} = D_t + |c_t| S0_{t+1} and
    S1_t = sum_k k |P_k| D_{t+k} = |c_t| (S1_{t+1} + S0_{t+1})."""
    c, D = np.abs(_d(coef)), _d(mag)
    N, T = D.shape
    s0, s1 = np.zeros(N), np.zeros(N)
    out = np.zeros((N, T))
    for t in range(T - 1, -1, -1):
        s1 = c[:, t] * (s1 + s0)
        s0 = D[:, t] + c[:, t] * s0
        out[:, t] = 2.0 * u * (s1 + L * s0)
    return out


def gae_mag(rew, val, seg_end, boot, gamma, use_gae=True):
    """D_t of gae_bound: |r_t| + gamma*|V'_t| + |V_t| for the GAE delta; |r_t| (+ gamma*|bootstrap_t| at a segment end)
    for the n-step returns."""
    r, v, b = np.abs(_d(rew)), np.abs(_d(val)), np.abs(_d(boot))
    se = np.asarray(seg_end) != 0
    g = f64(f32(gamma))
    vnext = np.where(se, b, np.concatenate([v[:, 1:], np.zeros((v.shape[0], 1))], axis=1))
    if use_gae:
        return r + g * vnext + v
    return np.where(se, r + g * b, r)


def ulp32(x):
    """The spacing of float32 at |x| (the gap to the next float32 away from zero)."""
    return np.spacing(np.abs(np.asarray(x, f64)).astype(f32)).astype(f64)


# ------------------------------------------------------------------------------------------------------ K10
def categorical(logits):
    """Categorical(logits) in float64: (lp, p, entropy, lse), entropy = -sum over p > 0 of p*lp (torch clamps the
    log-probabilities of zero-probability categories, so they add nothing; -inf logits stay finite)."""
    z = _d(logits)
    m = z.max(axis=1, keepdims=True)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        lse = m + np.log(np.exp(z - m).sum(axis=1, keepdims=True))
        lp = z - lse
        p = np.exp(lp)
        ent = -np.where(p > 0, p * lp, 0.0).sum(axis=1)
    return lp, p, ent, lse[:, 0]


def argmax_first(logits):
    """torch.argmax of the probabilities: the first maximal index (exp is monotone, so the first maximal logit)."""
    return np.argmax(_d(logits), axis=1)


def draw(p, u):
    """Inverse-CDF draw in float64: the first i with u < cdf_i; if no prefix passes u, the last index with p > 0."""
    p, u = _d(p), _d(u)
    cdf = np.cumsum(p, axis=1)
    hit = u[:, None] < cdf
    last_pos = p.shape[1] - 1 - np.argmax((p > 0)[:, ::-1], axis=1)
    return np.where(hit.any(axis=1), np.argmax(hit, axis=1), last_pos)


def categorical_bounds(logits):
    """Derived bounds for K10 in float32 (csrc/act.cu): (E [N,A], ent_bound [N], delta [N]).

    E_i bounds |lp32_i - lp_i|.  The kernel forms x_i = z_i - m (error <= u|x_i|), t_i = expf(x_i) (CUDA: <= 2 ulp,
    i.e. <= 4u relative; the error of x_i propagates as u|x_i| relative), se = t_0 + .. (sequential: <= (A-1)u * se),
    lse = m + logf(se) (logf <= 1 ulp, i.e. <= 2u |log se|; the addition <= u|lse|) and lp_i = z_i - lse (<= u|lp_i|).
    With se >= 1 (the maximal term is expf(0) = 1) and t|x| = e^x |x| <= 1/e, the relative error of se is at most
    (A - 1 + 4 + A/e) u and log se <= ln A, so
        E_i = u * (|lp_i| + |lse| + 2 ln A + (1 + 1/e) A + 3) * (1 + 2^-16)
    where the last factor covers the second-order terms (below 2 A u < 2^-16 for A <= 64).

    ent_bound: p32_i = expf(lp32_i) is within p_i (E_i + 4u) + 2 * 2^-149 of p_i (the lp error propagates as a
    relative error of p; 2 subnormal ulps in the underflow range), so each term p_i lp_i moves by at most
    p_i |lp_i| (E_i + 4u) + p_i E_i (+ the floor times |lp_i|), and forming and summing A terms adds at most
    A u sum_i p_i |lp_i|:  ent_bound = sum_i [p_i (|lp_i| (E_i + 4u + A u) + E_i) + 2^-148 |lp_i|] over finite lp_i.

    delta bounds |cdf32_i - cdf_i| for every i: the p errors above summed, plus the A sequential additions of
    probabilities whose partial sums are <= 1 + 2^-10: delta = sum_i (p_i (E_i + 4u) + 2^-148) + A u (1 + 2^-10).
    A draw is unambiguous when u is farther than delta from every cdf_i."""
    u = EPS32
    lp, p, _, lse = categorical(logits)
    A = lp.shape[1]
    fin = np.isfinite(lp)
    alp = np.where(fin, np.abs(lp), 0.0)
    E = u * (alp + np.abs(lse)[:, None] + 2 * np.log(A) + (1 + 1 / np.e) * A + 3) * (1 + 2.0 ** -16)
    ent_b = (p * (alp * (E + 4 * u + A * u) + E) + 2 * TINY32 * alp).sum(axis=1)
    delta = (p * (E + 4 * u) + 2 * TINY32).sum(axis=1) + A * u * (1 + 2.0 ** -10)
    return E, ent_b, delta


def draw_allowed(p, u, delta, a):
    """Whether action a[n] is consistent with an inverse-CDF draw over probabilities within delta[n] of p (the
    float32 kernel's): p_a > 0, and cdf_{a-1} - delta <= u < cdf_a + delta, or a is the last positive index and
    u >= cdf_{A-1} - delta (no prefix passed u)."""
    p, u, delta = _d(p), _d(u), _d(delta)
    N, A = p.shape
    a = np.asarray(a, np.int64)
    ok_idx = (a >= 0) & (a < A)
    a_c = np.clip(a, 0, A - 1)
    cdf = np.cumsum(p, axis=1)
    rows = np.arange(N)
    lo = np.where(a_c > 0, cdf[rows, a_c - 1], 0.0)
    hi = cdf[rows, a_c]
    last_pos = A - 1 - np.argmax((p > 0)[:, ::-1], axis=1)
    inside = (u >= lo - delta) & (u < hi + delta)
    tail = (a_c == last_pos) & (u >= cdf[:, -1] - delta)
    return ok_idx & (p[rows, a_c] > 0) & (inside | tail)


# ------------------------------------------------------------------------------------------------------ K11
def rms_update_f32(x, mean, var, count):
    """xb_rms_update_normalize's update in float32, in the header's operation order with the two column sums taken
    row after row.  Returns the new (mean, var)."""
    x = np.asarray(x, f32)
    N = x.shape[0]
    mean, var = np.asarray(mean, f32), np.asarray(var, f32)
    fn = f32(N)
    s = np.zeros(x.shape[1], f32)
    for n in range(N):
        s = s + x[n]
    bm = s / fn
    ss = np.zeros(x.shape[1], f32)
    for n in range(N):
        c = x[n] - bm
        ss = ss + c * c
    bstd = np.sqrt(ss / fn)
    bv = bstd * bstd
    cnt, tot = f32(count), f32(float(count) + N)
    delta = bm - mean
    new_mean = mean + (delta * fn) / tot
    m2 = (var * cnt + bv * fn) + (((delta * delta) * cnt) * fn) / tot
    return new_mean, m2 / tot


def rms_normalize_f32(x, mean, var, clip_range, eps=1e-8):
    """out = clip((x - mean) / (sqrt(var) + eps), -clip_range, clip_range) in float32."""
    denom = np.sqrt(np.asarray(var, f32)) + f32(eps)
    y = (np.asarray(x, f32) - np.asarray(mean, f32)) / denom
    return np.minimum(np.maximum(y, f32(-clip_range)), f32(clip_range))

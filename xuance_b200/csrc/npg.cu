// K4N fused NPG loss forward+backward (Categorical and DiagGaussian policies) and K7N, the closed-form natural gradient
// over the actor's flat gradient bucket.
//
// K4N runs one warp per row, lanes over the A actions / D action components (<= 64: two per lane).  Besides the loss
// seed of -mean(adv * log pi) it writes the score seed d(sum_b log pi_b) / d outputs, the critic seed and the fp64 sum of
// log pi that K7N reads.  Every reduction has a fixed order: the outputs are bit-identical from launch to launch.
//
// K7N rewrites each actor tensor's gradient g with (F^-1 g) for the reference's F = kappa s s^T + lam I
// (npg_learner.py:100-113), by Sherman-Morrison: F^-1 g = (g - s * kappa (s.g) / (lam + kappa s.s)) / lam.
#include "xb_common.cuh"

#define XB_NPG_CHUNK 4096   // K7N: elements per dot-product partial (one block of 256 threads, 16 per thread)
#define XB_LOG_SQRT_2PI_N 0.91893853320467274178f

static inline int npg_grid(int64_t B) {
    const int64_t want = (B + 7) / 8;  // 8 warps, one row each, per 256-thread block
    return (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
}

// stats[8] = {actor-loss, critic-loss, predict_value, sum log pi, 0, 0, 0, 0} from the fp64 sums
// {sum adv * log pi, sum (v - R)^2, sum v, sum log pi}; *logp_sum = the last one in fp64.
__device__ __forceinline__ void npg_write_stats(const double (&t)[4], int64_t B, float *stats, double *logp_sum) {
    const double ib = 1.0 / (double)B;
    stats[0] = (float)(-t[0] * ib);
    stats[1] = (float)(t[1] * ib);
    stats[2] = (float)(t[2] * ib);
    stats[3] = (float)t[3];
    stats[4] = 0.f;
    stats[5] = 0.f;
    stats[6] = 0.f;
    stats[7] = 0.f;
    *logp_sum = t[3];
}

// The value term of a row (lane 0): nn.MSELoss backward 2 (v - R) / B.
__device__ __forceinline__ void npg_value_row(int64_t b, const float *value, const float *ret, float norm,
                                              float *dvalue, double (&acc)[4]) {
    const float v = value[b], dv = __fsub_rn(v, ret[b]);
    dvalue[b] = __fmul_rn(norm, dv);
    acc[1] += (double)dv * (double)dv;
    acc[2] += (double)v;
}

// =====================================================================================================
// xb_npg_loss_fwd_bwd (Categorical)
// =====================================================================================================
// Categorical(logits=z): lp_i = z_i - logsumexp(z), p_i = exp(lp_i); log pi = lp_a.
//   score seed  d lp_a / d z_i = [i == a] - p_i;   loss seed  -(adv / B) ([i == a] - p_i).
__global__ void __launch_bounds__(256) npg_loss_kernel(const float *__restrict__ logits, const float *__restrict__ value,
                                                       const float *__restrict__ actions, const float *__restrict__ adv,
                                                       const float *__restrict__ ret, int64_t B, int A, float inv_b,
                                                       float *__restrict__ dlogits, float *__restrict__ dscore,
                                                       float *__restrict__ dvalue, float *__restrict__ stats,
                                                       double *__restrict__ logp_sum, double *__restrict__ scratch) {
    __shared__ double red[4 * 32];
    double acc[4] = {0, 0, 0, 0};  // sum adv * log pi, sum (v - R)^2, sum v, sum log pi
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const float norm = 2.f * inv_b;
    const bool h0 = lane < A, h1 = lane + 32 < A;
    for (int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < B; b += nw) {
        const float *zr = logits + b * A;
        const float z0 = h0 ? zr[lane] : -INFINITY, z1 = h1 ? zr[lane + 32] : -INFINITY;
        float m = fmaxf(z0, z1);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        const float se = warp_sum_f((h0 ? expf(z0 - m) : 0.f) + (h1 ? expf(z1 - m) : 0.f));
        const float lse = m + logf(se);
        const float lp0 = z0 - lse, lp1 = z1 - lse;
        const int a = (int)actions[b];
        const float lpa = __shfl_sync(0xffffffffu, a < 32 ? lp0 : lp1, a & 31);
        const float ad = adv[b];
        const float y0 = (lane == a ? 1.f : 0.f) - expf(lp0), y1 = (lane + 32 == a ? 1.f : 0.f) - expf(lp1);
        const float c = -ad * inv_b;
        if (h0) {
            dscore[b * A + lane] = y0;
            dlogits[b * A + lane] = c * y0;
        }
        if (h1) {
            dscore[b * A + lane + 32] = y1;
            dlogits[b * A + lane + 32] = c * y1;
        }
        if (lane == 0) {
            acc[0] += (double)(ad * lpa);
            acc[3] += (double)lpa;
            npg_value_row(b, value, ret, norm, dvalue, acc);
        }
    }
    grid_sum_finalize<4>(acc, scratch, red, [&](double(&t)[4]) { npg_write_stats(t, B, stats, logp_sum); });
}

extern "C" int xb_npg_loss_fwd_bwd(const float *logits, const float *value, const float *actions, const float *adv,
                                   const float *ret, int64_t B, int A, float *dlogits, float *dscore, float *dvalue,
                                   float *stats, double *logp_sum, double *scratch, void *stream) {
    if (!logits || !value || !actions || !adv || !ret || !dlogits || !dscore || !dvalue || !stats || !logp_sum ||
        !scratch)
        return XB_EINVAL;
    if (B <= 0 || A <= 0) return XB_EINVAL;
    if (A > 64) return XB_ERANGE;
    npg_loss_kernel<<<npg_grid(B), 256, 0, (cudaStream_t)stream>>>(logits, value, actions, adv, ret, B, A,
                                                                   1.0f / (float)B, dlogits, dscore, dvalue, stats,
                                                                   logp_sum, scratch);
    return xb_launch_status();
}

// =====================================================================================================
// xb_npg_gauss_loss_fwd_bwd (DiagGaussian)
// =====================================================================================================
// Normal(mu, exp(log_std)) summed over the D components, as K4G: with z_j = (x_j - mu_j) / sigma_j
//   log pi = sum_j (-z_j^2 / 2 - log_std_j - log sqrt(2 pi));  d log pi / d mu_j = z_j / sigma_j;
//   d log pi / d log_std_j = z_j^2 - 1.
// log_std is shared by every row: lane j of each warp owns columns j and j + 32 and adds its rows' terms in fp64; a block
// adds its 8 warps in warp order into ws[2][D][grid], and the last block to arrive adds those in block order.
__global__ void __launch_bounds__(256) npg_gauss_loss_kernel(
    const float *__restrict__ mu, const float *__restrict__ log_std, const float *__restrict__ value,
    const float *__restrict__ actions, const float *__restrict__ adv, const float *__restrict__ ret, int64_t B, int D,
    float inv_b, float *__restrict__ dmu, float *__restrict__ dlog_std, float *__restrict__ smu,
    float *__restrict__ slog_std, float *__restrict__ dvalue, float *__restrict__ stats, double *__restrict__ logp_sum,
    double *__restrict__ scratch, double *__restrict__ ws) {
    __shared__ double red[4 * 32];
    __shared__ double cred[2][64][8];  // [loss / score][column][warp]
    __shared__ float s_ls[64], s_isig[64];
    for (int j = threadIdx.x; j < D; j += blockDim.x) {
        const float ls = log_std[j];
        s_ls[j] = ls;
        s_isig[j] = 1.f / expf(ls);
    }
    __syncthreads();
    double acc[4] = {0, 0, 0, 0};
    double cl[2] = {0, 0}, cs[2] = {0, 0};  // this lane's columns (lane, lane + 32): loss and score sums
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const float norm = 2.f * inv_b;
    for (int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < B; b += nw) {
        const float c = -adv[b] * inv_b;
        float lp = 0.f;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int j = lane + 32 * k;
            if (j < D) {
                const float z = (actions[b * D + j] - mu[b * D + j]) * s_isig[j];
                lp += -0.5f * z * z - s_ls[j] - XB_LOG_SQRT_2PI_N;
                const float gm = z * s_isig[j], gl = z * z - 1.f;
                smu[b * D + j] = gm;
                dmu[b * D + j] = c * gm;
                cs[k] += (double)gl;
                cl[k] += (double)(c * gl);
            }
        }
        lp = warp_sum_f(lp);
        if (lane == 0) {
            acc[0] += (double)(adv[b] * lp);
            acc[3] += (double)lp;
            npg_value_row(b, value, ret, norm, dvalue, acc);
        }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int j = lane + 32 * k;
        if (j < D) {
            cred[0][j][warp] = cl[k];
            cred[1][j][warp] = cs[k];
        }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < 2 * D; t += blockDim.x) {
        const int w = t / D, j = t % D;
        double s = 0.0;
        for (int k = 0; k < 8; ++k) s += cred[w][j][k];
        ws[((int64_t)w * D + j) * gridDim.x + blockIdx.x] = s;
    }
    __threadfence();
    const bool last = grid_sum_finalize<4>(acc, scratch, red,
                                           [&](double(&t)[4]) { npg_write_stats(t, B, stats, logp_sum); });
    if (last) {
        for (int t = threadIdx.x; t < 2 * D; t += blockDim.x) {
            const double *p = ws + (int64_t)t * gridDim.x;
            double s = 0.0;
            for (int k = 0; k < (int)gridDim.x; ++k) s += __ldcg(&p[k]);
            if (t < D) dlog_std[t] = (float)s;
            else slog_std[t - D] = (float)s;
        }
    }
}

extern "C" int64_t xb_npg_gauss_ws_doubles(int64_t B, int D) {
    if (B <= 0 || D <= 0) return 0;
    return 2 * (int64_t)D * npg_grid(B);
}

extern "C" int xb_npg_gauss_loss_fwd_bwd(const float *mu, const float *log_std, const float *value,
                                         const float *actions, const float *adv, const float *ret, int64_t B, int D,
                                         float *dmu, float *dlog_std, float *smu, float *slog_std, float *dvalue,
                                         float *stats, double *logp_sum, double *scratch, double *ws,
                                         int64_t ws_doubles, void *stream) {
    if (!mu || !log_std || !value || !actions || !adv || !ret || !dmu || !dlog_std || !smu || !slog_std || !dvalue ||
        !stats || !logp_sum || !scratch || !ws)
        return XB_EINVAL;
    if (B <= 0 || D <= 0) return XB_EINVAL;
    if (D > 64) return XB_ERANGE;
    if (ws_doubles < xb_npg_gauss_ws_doubles(B, D)) return XB_EINVAL;
    npg_gauss_loss_kernel<<<npg_grid(B), 256, 0, (cudaStream_t)stream>>>(mu, log_std, value, actions, adv, ret, B, D,
                                                                         1.0f / (float)B, dmu, dlog_std, smu, slog_std,
                                                                         dvalue, stats, logp_sum, scratch, ws);
    return xb_launch_status();
}

// =====================================================================================================
// K7N  xb_npg_natural_grad
// =====================================================================================================
// table[3 * nseg] = {offset, length, first chunk} per segment (xb_npg_segment_table).  Pass 1: block c forms the fp64
// partials (s.g, s.s) of chunk c.  Pass 2: block c folds its segment's partials in chunk order (lane k takes chunks k,
// k + 32, ..., then a warp butterfly), forms the segment's coefficient and rewrites its chunk of g in place.
__device__ __forceinline__ int npg_segment_of(const int64_t *table, int nseg, int64_t c) {
    int lo = 0, hi = nseg - 1;  // the last segment whose first chunk is <= c
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (table[3 * mid + 2] <= c) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(256) npg_dot_kernel(const float *__restrict__ g, const float *__restrict__ s,
                                                      const int64_t *__restrict__ table, int nseg,
                                                      double *__restrict__ ws) {
    __shared__ double red[2 * 32];
    const int64_t c = blockIdx.x;
    const int i = npg_segment_of(table, nseg, c);
    const int64_t off = table[3 * i], len = table[3 * i + 1];
    const int64_t lo = (c - table[3 * i + 2]) * XB_NPG_CHUNK;
    const int64_t hi = min(lo + (int64_t)XB_NPG_CHUNK, len);
    double v[2] = {0.0, 0.0};  // s.g, s.s
    for (int64_t k = lo + threadIdx.x; k < hi; k += blockDim.x) {
        const double sk = (double)s[off + k];
        v[0] += sk * (double)g[off + k];
        v[1] += sk * sk;
    }
    block_sum_d<2>(v, red);
    if (threadIdx.x == 0) {
        ws[2 * c] = v[0];
        ws[2 * c + 1] = v[1];
    }
}

__global__ void __launch_bounds__(256) npg_apply_kernel(float *__restrict__ g, const float *__restrict__ s,
                                                        const int64_t *__restrict__ table, int nseg,
                                                        const double *__restrict__ ws,
                                                        const double *__restrict__ logp_sum, double horizon,
                                                        double lam) {
    __shared__ double coef;
    const int64_t c = blockIdx.x;
    const int i = npg_segment_of(table, nseg, c);
    const int64_t off = table[3 * i], len = table[3 * i + 1], first = table[3 * i + 2];
    if (threadIdx.x < 32) {
        const int64_t n = (len + XB_NPG_CHUNK - 1) / XB_NPG_CHUNK;
        double sg = 0.0, ss = 0.0;
        for (int64_t k = threadIdx.x; k < n; k += 32) {
            sg += ws[2 * (first + k)];
            ss += ws[2 * (first + k) + 1];
        }
        sg = warp_sum_d(sg);
        ss = warp_sum_d(ss);
        if (threadIdx.x == 0) {
            const double kappa = *logp_sum / horizon;
            coef = kappa * sg / (lam + kappa * ss);  // no guard: F is singular there, as the reference's inverse is
        }
    }
    __syncthreads();
    const double cf = coef, inv_lam = 1.0 / lam;
    const int64_t lo = (c - first) * XB_NPG_CHUNK;
    const int64_t hi = min(lo + (int64_t)XB_NPG_CHUNK, len);
    for (int64_t k = lo + threadIdx.x; k < hi; k += blockDim.x)
        g[off + k] = (float)(((double)g[off + k] - (double)s[off + k] * cf) * inv_lam);
}

extern "C" int64_t xb_npg_segment_table(const int64_t *offsets, const int64_t *lengths, int nseg, int64_t *table) {
    if (!offsets || !lengths || !table || nseg <= 0) return XB_EINVAL;
    int64_t chunks = 0;
    for (int i = 0; i < nseg; ++i) {
        if (offsets[i] < 0 || lengths[i] <= 0) return XB_EINVAL;
        table[3 * i] = offsets[i];
        table[3 * i + 1] = lengths[i];
        table[3 * i + 2] = chunks;
        chunks += (lengths[i] + XB_NPG_CHUNK - 1) / XB_NPG_CHUNK;
    }
    return chunks;
}

extern "C" int xb_npg_natural_grad(float *g, const float *s, const int64_t *table, int nseg, int64_t nchunks,
                                   const double *logp_sum, double horizon, double lam, double *ws, int64_t ws_doubles,
                                   void *stream) {
    if (!g || !s || !table || !logp_sum || !ws) return XB_EINVAL;
    if (nseg <= 0 || nchunks < nseg || !(horizon > 0.0) || !(lam > 0.0)) return XB_EINVAL;
    if (nchunks > 0x7fffffffLL) return XB_ERANGE;
    if (ws_doubles < 2 * nchunks) return XB_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    npg_dot_kernel<<<(unsigned)nchunks, 256, 0, st>>>(g, s, table, nseg, ws);
    npg_apply_kernel<<<(unsigned)nchunks, 256, 0, st>>>(g, s, table, nseg, ws, logp_sum, horizon, lam);
    return xb_launch_status();
}

// =====================================================================================================
// K6Z  C51 / QR-DQN (xuance/torch/learners/qlearning_family/{c51,qrdqn}_learner.py, deep_q_network.py:146-325)
// =====================================================================================================
// xb_dist_greedy: the no-grad head tail of C51DeepQNetwork / QRDeepQNetwork (softmax, expected Q, argmax).
// xb_c51_loss_fwd_bwd / xb_qrdqn_loss_fwd_bwd: the whole loss of each learner and its autograd to the eval head's
// raw [B, A, N] output, in one launch.  One warp per row b; lane l owns atoms l and l + 32 (N <= 64).  All three
// entry points share dist_row_greedy for the softmax, the expected Q and the argmax, so the loss kernels' target
// action is exactly the action xb_dist_greedy returns for the same tensor.  The float32 arithmetic that is meant to
// match torch bit for bit (C51's Tz and projection weights, QR's backup) is written with explicit _rn intrinsics in
// torch's evaluation order.  Statistics are float64 partial sums through grid_sum_finalize: no float atomics.
#include "xb_common.cuh"

#define K6Z_MAX_N 64
#define K6Z_MAX_A 256
#define K6Z_ROWS_PER_BLOCK 8   // 256 threads, one warp per row

// torch.clamp / maximum / minimum: a NaN operand is the result (fmaxf / fminf would drop it)
__device__ __forceinline__ float k6z_maxn(float a, float b) { return a != a ? a : (b != b ? b : fmaxf(a, b)); }
__device__ __forceinline__ float k6z_minn(float a, float b) { return a != a ? a : (b != b ? b : fminf(a, b)); }
__device__ __forceinline__ float k6z_clamp(float x, float lo, float hi) { return k6z_minn(k6z_maxn(x, lo), hi); }

// xor butterflies: float addition and max are commutative, so every lane ends with the bit-identical result
__device__ __forceinline__ float k6z_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float k6z_warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = k6z_maxn(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

struct DistRow {
    float x0, x1;  // this lane's two atoms: softmax probabilities (C51) or raw quantiles (QR); 0 past N
};

// Softmax of one C51 action row in float32: m = max_i x_i; e_i = expf(x_i - m); s = sum_i e_i (lane partials, then
// the xor butterfly); p_i = e_i / s (correctly rounded division).  Every lane returns its two p.
__device__ __forceinline__ DistRow k6z_softmax(const float *__restrict__ x, int N, int lane) {
    const bool h0 = lane < N, h1 = lane + 32 < N;
    const float v0 = h0 ? x[lane] : -INFINITY, v1 = h1 ? x[lane + 32] : -INFINITY;
    const float m = k6z_warp_max(k6z_maxn(v0, v1));
    const float e0 = h0 ? expf(__fsub_rn(v0, m)) : 0.f, e1 = h1 ? expf(__fsub_rn(v1, m)) : 0.f;
    const float s = k6z_warp_sum(__fadd_rn(e0, e1));
    return DistRow{h0 ? __fdiv_rn(e0, s) : 0.f, h1 ? __fdiv_rn(e1, s) : 0.f};
}

// The shared head tail.  For each action a of row `z` ([A, N]): C51 (supports != NULL) takes p = softmax(z[a]) and
// Q_a = sum_i supports_i * p_i; QR takes Q_a = (sum_i z[a, i]) / N.  The sums are lane partials (atom l, then l + 32)
// reduced by the xor butterfly.  The argmax is the FIRST maximal index, as torch.argmax chooses, and a NaN Q wins
// (torch.argmax treats NaN as the maximum).  Optionally writes q[A] and probs[A, N]; returns the greedy action and
// leaves its row (probabilities or quantiles) in `best`.
__device__ __forceinline__ int dist_row_greedy(const float *__restrict__ z, const float *__restrict__ supports, int A,
                                               int N, int lane, DistRow &best, float *__restrict__ q,
                                               float *__restrict__ probs) {
    const bool h0 = lane < N, h1 = lane + 32 < N;
    const float s0 = (supports && h0) ? supports[lane] : 0.f, s1 = (supports && h1) ? supports[lane + 32] : 0.f;
    int best_a = 0;
    float best_q = 0.f;
    best = DistRow{0.f, 0.f};
    for (int a = 0; a < A; ++a) {
        const float *row = z + (int64_t)a * N;
        DistRow r;
        float qa;
        if (supports) {
            r = k6z_softmax(row, N, lane);
            qa = k6z_warp_sum(__fadd_rn(__fmul_rn(s0, r.x0), __fmul_rn(s1, r.x1)));
            if (probs) {
                if (h0) probs[(int64_t)a * N + lane] = r.x0;
                if (h1) probs[(int64_t)a * N + lane + 32] = r.x1;
            }
        } else {
            r = DistRow{h0 ? row[lane] : 0.f, h1 ? row[lane + 32] : 0.f};
            qa = __fdiv_rn(k6z_warp_sum(__fadd_rn(r.x0, r.x1)), (float)N);
        }
        if (q && lane == 0) q[a] = qa;
        const bool take = a == 0 || (best_q == best_q && (qa != qa || qa > best_q));
        if (take) {
            best_a = a;
            best_q = qa;
            best = r;
        }
    }
    return best_a;
}

static inline int k6z_grid(int64_t rows) {
    const int64_t want = (rows + K6Z_ROWS_PER_BLOCK - 1) / K6Z_ROWS_PER_BLOCK;
    return (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
}

static inline bool k6z_shape_ok(int64_t B, int A, int N) {
    return B > 0 && A >= 1 && A <= K6Z_MAX_A && N >= 2 && N <= K6Z_MAX_N;
}

// -------------------------------------------------------------------------------------------- xb_dist_greedy
__global__ void __launch_bounds__(256) dist_greedy_kernel(const float *__restrict__ z,
                                                          const float *__restrict__ supports, int64_t B, int A, int N,
                                                          int64_t *__restrict__ actions, float *__restrict__ q,
                                                          float *__restrict__ probs) {
    const int lane = threadIdx.x & 31;
    const int64_t wstride = (int64_t)gridDim.x * K6Z_ROWS_PER_BLOCK;
    for (int64_t b = (int64_t)blockIdx.x * K6Z_ROWS_PER_BLOCK + (threadIdx.x >> 5); b < B; b += wstride) {
        DistRow best;
        const int a = dist_row_greedy(z + b * A * N, supports, A, N, lane, best, q ? q + b * A : nullptr,
                                      probs ? probs + b * A * N : nullptr);
        if (lane == 0) actions[b] = a;
    }
}

extern "C" int xb_dist_greedy(const float *z, const float *supports, int64_t B, int A, int N, int64_t *actions,
                              float *q, float *probs, void *stream) {
    if (!z || !actions) return XB_EINVAL;
    if (!k6z_shape_ok(B, A, N)) return XB_EINVAL;
    if (probs && !supports) return XB_EINVAL;  // probabilities exist for C51 only
    dist_greedy_kernel<<<k6z_grid(B), 256, 0, (cudaStream_t)stream>>>(z, supports, B, A, N, actions, q, probs);
    return xb_launch_status();
}

// -------------------------------------------------------------------------------------------- xb_c51_loss_fwd_bwd
// c51_learner.py:42-51.  Per row: the target network's greedy action a' and its probabilities p'_j (dist_row_greedy);
// Tz_j = clamp(rew + (gamma*z_j)*(1 - ter), v_min, v_max); w_ji = clamp(1 - |Tz_j - z_i| / dz, 0, 1);
// target_i = sum_j p'_j * w_ji accumulated in float32 from j = 0 up (lane i; p'_j and Tz_j broadcast by shuffle);
// p = softmax(eval[a]); loss_b = -sum_i target_i * log(p_i + 1e-8); dlogits[a] = p * (g - sum_i p_i g_i) with
// g_i = ((-1/B_total) * target_i) / (p_i + 1e-8), the other actions' rows 0.
__global__ void __launch_bounds__(256) c51_loss_kernel(
    const float *__restrict__ z_eval, const float *__restrict__ z_next, const float *__restrict__ supports,
    const float *__restrict__ actions, const float *__restrict__ rew, const float *__restrict__ ter, int64_t B, int A,
    int N, float gamma, float v_min, float v_max, float dz, float seed, float *__restrict__ dlogits,
    int64_t *__restrict__ target_actions, float *__restrict__ target_dist, float *__restrict__ stats,
    double *__restrict__ scratch, float inv_bt) {
    __shared__ double red[32];
    double acc[1] = {0};
    const int lane = threadIdx.x & 31;
    const bool h0 = lane < N, h1 = lane + 32 < N;
    const float zi0 = h0 ? supports[lane] : 0.f, zi1 = h1 ? supports[lane + 32] : 0.f;
    const float gz0 = __fmul_rn(gamma, zi0), gz1 = __fmul_rn(gamma, zi1);
    const int64_t wstride = (int64_t)gridDim.x * K6Z_ROWS_PER_BLOCK;
    for (int64_t b = (int64_t)blockIdx.x * K6Z_ROWS_PER_BLOCK + (threadIdx.x >> 5); b < B; b += wstride) {
        DistRow pt;
        const int ta = dist_row_greedy(z_next + b * A * N, supports, A, N, lane, pt, nullptr, nullptr);
        if (lane == 0) target_actions[b] = ta;
        // next_supports = rew + (gamma * supports) * (1 - ter), then clamp: torch's order (c51_learner.py:46-47)
        const float nt = __fsub_rn(1.f, ter[b]), r = rew[b];
        const float tz0 = k6z_clamp(__fadd_rn(r, __fmul_rn(gz0, nt)), v_min, v_max);
        const float tz1 = k6z_clamp(__fadd_rn(r, __fmul_rn(gz1, nt)), v_min, v_max);
        float t0 = 0.f, t1 = 0.f;
        for (int j = 0; j < N; ++j) {
            const int src = j & 31;
            const float pj = __shfl_sync(0xffffffffu, j < 32 ? pt.x0 : pt.x1, src);
            const float tzj = __shfl_sync(0xffffffffu, j < 32 ? tz0 : tz1, src);
            const float w0 = k6z_clamp(__fsub_rn(1.f, __fdiv_rn(fabsf(__fsub_rn(tzj, zi0)), dz)), 0.f, 1.f);
            const float w1 = k6z_clamp(__fsub_rn(1.f, __fdiv_rn(fabsf(__fsub_rn(tzj, zi1)), dz)), 0.f, 1.f);
            t0 = __fadd_rn(t0, __fmul_rn(pj, w0));
            t1 = __fadd_rn(t1, __fmul_rn(pj, w1));
        }
        if (target_dist) {
            if (h0) target_dist[b * N + lane] = t0;
            if (h1) target_dist[b * N + lane + 32] = t1;
        }
        // the eval side: only the taken action's row has a gradient.  An action outside [0, A) selects no row: its
        // gradient is 0 and it adds NaN to the loss, so a corrupt batch shows without an out-of-bounds read.
        const float af = actions[b];
        const int a = (af >= 0.f && af < (float)A) ? (int)af : -1;
        float *g = dlogits + b * A * N;
        for (int i = lane; i < A * N; i += 32)
            if (i < a * N || i >= (a + 1) * N) g[i] = 0.f;
        if (a < 0) {
            if (lane == 0) acc[0] += (double)NAN;
            continue;
        }
        const DistRow p = k6z_softmax(z_eval + (b * A + a) * N, N, lane);
        const float q0 = __fadd_rn(p.x0, 1e-8f), q1 = __fadd_rn(p.x1, 1e-8f);
        float l = 0.f;
        if (h0) l = __fmul_rn(t0, logf(q0));
        if (h1) l = __fadd_rn(l, __fmul_rn(t1, logf(q1)));
        acc[0] -= (double)l;
        const float g0 = h0 ? __fdiv_rn(__fmul_rn(seed, t0), q0) : 0.f;
        const float g1 = h1 ? __fdiv_rn(__fmul_rn(seed, t1), q1) : 0.f;
        const float dot = k6z_warp_sum(__fadd_rn(__fmul_rn(p.x0, g0), __fmul_rn(p.x1, g1)));
        if (h0) g[a * N + lane] = __fmul_rn(p.x0, __fsub_rn(g0, dot));
        if (h1) g[a * N + lane + 32] = __fmul_rn(p.x1, __fsub_rn(g1, dot));
    }
    grid_sum_finalize<1>(acc, scratch, red, [&](double(&s)[1]) {
        stats[0] = (float)(s[0] * (double)inv_bt);  // Qloss
        stats[1] = stats[2] = stats[3] = 0.f;
    });
}

extern "C" int xb_c51_loss_fwd_bwd(const float *z_eval, const float *z_next, const float *supports,
                                   const float *actions, const float *rew, const float *ter, int64_t B, int A, int N,
                                   int64_t B_total, float gamma, float v_min, float v_max, float delta_z,
                                   float *dlogits, int64_t *target_actions, float *target_dist, float *stats,
                                   double *scratch, void *stream) {
    if (!z_eval || !z_next || !supports || !actions || !rew || !ter || !dlogits || !target_actions || !stats ||
        !scratch)
        return XB_EINVAL;
    if (!k6z_shape_ok(B, A, N) || B_total < B) return XB_EINVAL;
    const float inv_bt = 1.0f / (float)B_total;
    // autograd's seed: mean's backward is 1/numel (float32), then the negation
    const float seed = -(1.0f / (float)B_total);
    c51_loss_kernel<<<k6z_grid(B), 256, 0, (cudaStream_t)stream>>>(z_eval, z_next, supports, actions, rew, ter, B, A,
                                                                   N, gamma, v_min, v_max, delta_z, seed, dlogits,
                                                                   target_actions, target_dist, stats, scratch,
                                                                   inv_bt);
    return xb_launch_status();
}

// -------------------------------------------------------------------------------------------- xb_qrdqn_loss_fwd_bwd
// qrdqn_learner.py:44-48.  Per row: the target network's greedy action a' by mean(quantiles) (dist_row_greedy);
// y_j = rew + (gamma*theta'_j)*(1 - ter); loss = mse(y, theta[a]) over B_total*N; dq[a] = 2*(theta - y)/(B_total*N),
// the other actions' rows 0.
__global__ void __launch_bounds__(256) qrdqn_loss_kernel(
    const float *__restrict__ z_eval, const float *__restrict__ z_next, const float *__restrict__ actions,
    const float *__restrict__ rew, const float *__restrict__ ter, int64_t B, int A, int N, float gamma, float scale,
    float *__restrict__ dq, int64_t *__restrict__ target_actions, float *__restrict__ stats,
    double *__restrict__ scratch, double inv_n) {
    __shared__ double red[32];
    double acc[1] = {0};
    const int lane = threadIdx.x & 31;
    const bool h0 = lane < N, h1 = lane + 32 < N;
    const int64_t wstride = (int64_t)gridDim.x * K6Z_ROWS_PER_BLOCK;
    for (int64_t b = (int64_t)blockIdx.x * K6Z_ROWS_PER_BLOCK + (threadIdx.x >> 5); b < B; b += wstride) {
        DistRow th;
        const int ta = dist_row_greedy(z_next + b * A * N, nullptr, A, N, lane, th, nullptr, nullptr);
        if (lane == 0) target_actions[b] = ta;
        // rew + (gamma * target_quantile) * (1 - ter): torch's order (qrdqn_learner.py:46)
        const float nt = __fsub_rn(1.f, ter[b]), r = rew[b];
        const float y0 = __fadd_rn(r, __fmul_rn(__fmul_rn(gamma, th.x0), nt));
        const float y1 = __fadd_rn(r, __fmul_rn(__fmul_rn(gamma, th.x1), nt));
        const float af = actions[b];
        const int a = (af >= 0.f && af < (float)A) ? (int)af : -1;
        float *g = dq + b * A * N;
        for (int i = lane; i < A * N; i += 32)
            if (i < a * N || i >= (a + 1) * N) g[i] = 0.f;
        if (a < 0) {
            if (lane == 0) acc[0] += (double)NAN;
            continue;
        }
        const float *x = z_eval + (b * A + a) * N;
        if (h0) {
            const float e = __fsub_rn(x[lane], y0);
            acc[0] += (double)e * e;
            g[a * N + lane] = __fmul_rn(e, scale);
        }
        if (h1) {
            const float e = __fsub_rn(x[lane + 32], y1);
            acc[0] += (double)e * e;
            g[a * N + lane + 32] = __fmul_rn(e, scale);
        }
    }
    grid_sum_finalize<1>(acc, scratch, red, [&](double(&s)[1]) {
        stats[0] = (float)(s[0] * inv_n);  // Qloss
        stats[1] = stats[2] = stats[3] = 0.f;
    });
}

extern "C" int xb_qrdqn_loss_fwd_bwd(const float *z_eval, const float *z_next, const float *actions, const float *rew,
                                     const float *ter, int64_t B, int A, int N, int64_t B_total, float gamma,
                                     float *dq, int64_t *target_actions, float *stats, double *scratch, void *stream) {
    if (!z_eval || !z_next || !actions || !rew || !ter || !dq || !target_actions || !stats || !scratch)
        return XB_EINVAL;
    if (!k6z_shape_ok(B, A, N) || B_total < B) return XB_EINVAL;
    const double n = (double)B_total * (double)N;
    const float scale = (float)(2.0 / n);
    qrdqn_loss_kernel<<<k6z_grid(B), 256, 0, (cudaStream_t)stream>>>(z_eval, z_next, actions, rew, ter, B, A, N, gamma,
                                                                     scale, dq, target_actions, stats, scratch,
                                                                     1.0 / n);
    return xb_launch_status();
}

// K4P fused PPG auxiliary-phase loss forward+backward (Categorical and DiagGaussian policies).
// One warp per row, lanes over the A actions / D action components (<= 64: two per lane), warp butterflies for the row
// reductions, fp64 grid sums of the logged statistics: every output is bit-identical from launch to launch.
#include "xb_common.cuh"

__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// torch.logsumexp(dim=-1, keepdim=True) over the lanes' (x0, x1): an infinite max is replaced by 0 before the shift.
__device__ __forceinline__ float warp_logsumexp(float x0, float x1, bool h0, bool h1) {
    float m = warp_max_f(fmaxf(h0 ? x0 : -INFINITY, h1 ? x1 : -INFINITY));
    if (fabsf(m) == INFINITY) m = 0.f;
    const float s = warp_sum_f((h0 ? expf(x0 - m) : 0.f) + (h1 ? expf(x1 - m) : 0.f));
    return logf(s) + m;
}

// torch.softmax(dim=-1) of the lanes' (x0, x1) into (p0, p1).
__device__ __forceinline__ void warp_softmax(float x0, float x1, bool h0, bool h1, float &p0, float &p1) {
    const float m = warp_max_f(fmaxf(h0 ? x0 : -INFINITY, h1 ? x1 : -INFINITY));
    const float e0 = h0 ? expf(x0 - m) : 0.f, e1 = h1 ? expf(x1 - m) : 0.f;
    const float s = warp_sum_f(e0 + e1);
    p0 = e0 / s;
    p1 = e1 / s;
}

// The statistics every K4P launch logs, from the fp64 sums {sum (v-aux)^2, sum KL, sum (v-R)^2, sum v}; kl_div is the
// number of KL terms per row the mean runs over (1 Categorical, D Gaussian).
__device__ __forceinline__ void ppg_write_stats(const double (&t)[4], double inv_bt, int kl_div, float kl_beta,
                                                float *stats) {
    const float aux = (float)(t[0] * inv_bt), kl = (float)(t[1] * inv_bt / (double)kl_div);
    const float val = (float)(t[2] * inv_bt);
    stats[0] = aux;
    stats[1] = kl;
    stats[2] = val;
    stats[3] = __fadd_rn(__fadd_rn(aux, __fmul_rn(kl_beta, kl)), val);  // aux_loss + kl_beta * kl_loss + value_loss
    stats[4] = (float)(t[3] * inv_bt);
    stats[5] = 0.f;
    stats[6] = 0.f;
    stats[7] = 0.f;
}

// The value terms of a row (lane 0): value_loss = MSE(v, R) and aux_loss = MSE(v.detach(), aux_v).  nn.MSELoss backward
// is (2 / N) * (input - target), and the target's gradient its negative.
__device__ __forceinline__ void ppg_value_row(int64_t b, const float *value, const float *aux_value, const float *ret,
                                              float norm, float *dvalue, float *daux, double (&acc)[4]) {
    const float v = value[b], dv = __fsub_rn(v, ret[b]);
    dvalue[b] = __fmul_rn(norm, dv);
    acc[2] += (double)dv * (double)dv;
    acc[3] += (double)v;
    if (aux_value) {
        const float da = __fsub_rn(v, aux_value[b]);
        daux[b] = -__fmul_rn(norm, da);
        acc[0] += (double)da * (double)da;
    }
}

// =====================================================================================================
// xb_ppg_aux_loss_fwd_bwd (Categorical)
// =====================================================================================================
// ppg_learner.py:127-131 for a CategoricalDistribution, and its autograd backward down to (logits, value, aux_value).
// KL(new || old) is torch's _kl_categorical_categorical on Categorical(logits=z) and Categorical(logits=o):
//   lp = z - logsumexp(z), p = softmax(lp) (likewise lq, q);  t_i = p_i * (lp_i - lq_i);  t_i = inf where q_i == 0;
//   t_i = 0 where p_i == 0;  KL = sum_i t_i.
// The backward is autograd's, term by term, with c = kl_beta / B_total the upstream gradient of each row's KL:
//   g_i = 0 where the index_put masks wrote (p_i == 0 or q_i == 0), else c
//   dp_i = g_i * (lp_i - lq_i)                     (0 * inf = NaN: a -inf logit on either side makes the row NaN,
//                                                   as in torch)
//   dlp_i = p_i * (dp_i - sum_k p_k dp_k) + g_i * p_i                (softmax backward + the direct product term)
//   dz_j = dlp_j - exp(z_j - logsumexp(z)) * sum_k dlp_k             (log_softmax through logsumexp)
template <bool POLICY>
__global__ void __launch_bounds__(256) ppg_aux_kernel(const float *__restrict__ logits, const float *__restrict__ old_logits,
                                                      const float *__restrict__ value, const float *__restrict__ aux_value,
                                                      const float *__restrict__ ret, int64_t B, int A, float inv_bt,
                                                      float c, float kl_beta, float *__restrict__ dlogits,
                                                      float *__restrict__ dvalue, float *__restrict__ daux,
                                                      float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[4 * 32];
    double acc[4] = {0, 0, 0, 0};  // sum (v - aux)^2, sum KL, sum (v - R)^2, sum v
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const float norm = 2.f * inv_bt;
    const bool h0 = lane < A, h1 = lane + 32 < A;
    for (int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < B; b += nw) {
        if (POLICY) {
            const float *zr = logits + b * A, *orow = old_logits + b * A;
            const float z0 = h0 ? zr[lane] : 0.f, z1 = h1 ? zr[lane + 32] : 0.f;
            const float o0 = h0 ? orow[lane] : 0.f, o1 = h1 ? orow[lane + 32] : 0.f;
            const float lse_p = warp_logsumexp(z0, z1, h0, h1), lse_q = warp_logsumexp(o0, o1, h0, h1);
            const float lp0 = z0 - lse_p, lp1 = z1 - lse_p, lq0 = o0 - lse_q, lq1 = o1 - lse_q;
            float p0, p1, q0, q1;
            warp_softmax(lp0, lp1, h0, h1, p0, p1);
            warp_softmax(lq0, lq1, h0, h1, q0, q1);
            const float d0 = lp0 - lq0, d1 = lp1 - lq1;
            const float t0 = p0 == 0.f ? 0.f : (q0 == 0.f ? INFINITY : p0 * d0);
            const float t1 = p1 == 0.f ? 0.f : (q1 == 0.f ? INFINITY : p1 * d1);
            acc[1] += (h0 ? (double)t0 : 0.0) + (h1 ? (double)t1 : 0.0);
            const float g0 = (p0 == 0.f || q0 == 0.f) ? 0.f : c, g1 = (p1 == 0.f || q1 == 0.f) ? 0.f : c;
            const float dp0 = g0 * d0, dp1 = g1 * d1;
            const float s1 = warp_sum_f((h0 ? p0 * dp0 : 0.f) + (h1 ? p1 * dp1 : 0.f));
            const float G0 = p0 * (dp0 - s1) + g0 * p0, G1 = p1 * (dp1 - s1) + g1 * p1;
            const float sg = warp_sum_f((h0 ? G0 : 0.f) + (h1 ? G1 : 0.f));
            float *dz = dlogits + b * A;
            if (h0) dz[lane] = G0 - expf(z0 - lse_p) * sg;
            if (h1) dz[lane + 32] = G1 - expf(z1 - lse_p) * sg;
        }
        if (lane == 0) ppg_value_row(b, value, aux_value, ret, norm, dvalue, daux, acc);
    }
    grid_sum_finalize<4>(acc, scratch, red,
                         [&](double(&t)[4]) { ppg_write_stats(t, (double)inv_bt, 1, kl_beta, stats); });
}

static inline int ppg_grid(int64_t B) {
    const int64_t want = (B + 7) / 8;  // 8 warps, one row each, per 256-thread block
    return (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
}

extern "C" int xb_ppg_aux_loss_fwd_bwd(const float *logits, const float *old_logits, const float *value,
                                       const float *aux_value, const float *ret, int64_t B, int A, int64_t B_total,
                                       float kl_beta, float *dlogits, float *dvalue, float *daux, float *stats,
                                       double *scratch, void *stream) {
    if (!value || !ret || !dvalue || !stats || !scratch) return XB_EINVAL;
    const bool policy = logits != nullptr;
    if ((old_logits != nullptr) != policy || (dlogits != nullptr) != policy) return XB_EINVAL;
    if ((aux_value != nullptr) != (daux != nullptr)) return XB_EINVAL;
    if (B <= 0 || B_total < B) return XB_EINVAL;
    if (policy && A <= 0) return XB_EINVAL;
    if (policy && A > 64) return XB_ERANGE;
    const float inv_bt = 1.0f / (float)B_total;
    const float c = kl_beta / (float)B_total;  // MeanBackward of kl_beta * KL.mean()
    cudaStream_t s = (cudaStream_t)stream;
    if (policy)
        ppg_aux_kernel<true><<<ppg_grid(B), 256, 0, s>>>(logits, old_logits, value, aux_value, ret, B, A, inv_bt, c,
                                                         kl_beta, dlogits, dvalue, daux, stats, scratch);
    else
        ppg_aux_kernel<false><<<ppg_grid(B), 256, 0, s>>>(nullptr, nullptr, value, aux_value, ret, B, 0, inv_bt, c,
                                                          kl_beta, nullptr, dvalue, daux, stats, scratch);
    return xb_launch_status();
}

// =====================================================================================================
// xb_ppg_aux_gauss_loss_fwd_bwd (DiagGaussian)
// =====================================================================================================
// ppg_learner.py:127-131 for a DiagGaussianDistribution: a plain Normal(mu, exp(log_std)) against Normal(old_mu,
// exp(old_log_std)), so KL is [B, D] (torch's _kl_normal_normal) and .mean() runs over B * D terms:
//   vr = (s / so)^2, x = (mu - old_mu) / so, KL = 0.5 * (vr + x^2 - 1 - log vr),   s = exp(log_std), so = exp(old_log_std)
// With c = kl_beta / (B_total * D) and h = 0.5 c, autograd gives per term
//   dmu = h * (2 x) / so,   d log_std (one term) = ((h - h / vr) * (2 r) / so) * s,   r = s / so.
// The log_std term depends on the column alone (both scales are shared by every row), so the sum over the B local rows
// that the broadcast backward takes is B times it, formed in double: no cross-row reduction, bit-identical by
// construction.
template <int D_MAX>
__global__ void __launch_bounds__(256) ppg_aux_gauss_kernel(
    const float *__restrict__ mu, const float *__restrict__ log_std, const float *__restrict__ old_mu,
    const float *__restrict__ old_log_std, const float *__restrict__ value, const float *__restrict__ aux_value,
    const float *__restrict__ ret, int64_t B, int D, float inv_bt, float c, float kl_beta, float *__restrict__ dmu,
    float *__restrict__ dlog_std, float *__restrict__ dvalue, float *__restrict__ daux, float *__restrict__ stats,
    double *__restrict__ scratch) {
    __shared__ double red[4 * 32];
    __shared__ float s_so[D_MAX], s_vr[D_MAX], s_lvr[D_MAX];
    const float h = 0.5f * c;
    for (int j = threadIdx.x; j < D; j += blockDim.x) {
        const float sj = expf(log_std[j]), so = expf(old_log_std[j]);
        const float r = sj / so, vr = r * r;
        s_so[j] = so;
        s_vr[j] = vr;
        s_lvr[j] = logf(vr);
        if (blockIdx.x == 0) {
            const float g = (((h - h / vr) * (2.f * r)) / so) * sj;
            dlog_std[j] = (float)((double)B * (double)g);
        }
    }
    __syncthreads();
    double acc[4] = {0, 0, 0, 0};
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const float norm = 2.f * inv_bt;
    for (int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < B; b += nw) {
#pragma unroll
        for (int k = 0; k < (D_MAX + 31) / 32; ++k) {
            const int j = lane + 32 * k;
            if (j < D) {
                const float so = s_so[j], vr = s_vr[j];
                const float x = (mu[b * D + j] - old_mu[b * D + j]) / so;
                const float kl = 0.5f * (((vr + x * x) - 1.f) - s_lvr[j]);
                acc[1] += (double)kl;
                dmu[b * D + j] = (h * (2.f * x)) / so;
            }
        }
        if (lane == 0) ppg_value_row(b, value, aux_value, ret, norm, dvalue, daux, acc);
    }
    grid_sum_finalize<4>(acc, scratch, red,
                         [&](double(&t)[4]) { ppg_write_stats(t, (double)inv_bt, D, kl_beta, stats); });
}

extern "C" int xb_ppg_aux_gauss_loss_fwd_bwd(const float *mu, const float *log_std, const float *old_mu,
                                             const float *old_log_std, const float *value, const float *aux_value,
                                             const float *ret, int64_t B, int D, int64_t B_total, float kl_beta,
                                             float *dmu, float *dlog_std, float *dvalue, float *daux, float *stats,
                                             double *scratch, void *stream) {
    if (!mu || !log_std || !old_mu || !old_log_std || !value || !aux_value || !ret || !dmu || !dlog_std || !dvalue ||
        !daux || !stats || !scratch)
        return XB_EINVAL;
    if (B <= 0 || B_total < B || D <= 0) return XB_EINVAL;
    if (D > 64) return XB_ERANGE;
    const float inv_bt = 1.0f / (float)B_total;
    const float c = kl_beta / (float)((double)B_total * (double)D);  // MeanBackward over B_total * D terms
    cudaStream_t s = (cudaStream_t)stream;
#define XB_PPGG(DM)                                                                                                  \
    ppg_aux_gauss_kernel<DM><<<ppg_grid(B), 256, 0, s>>>(mu, log_std, old_mu, old_log_std, value, aux_value, ret, B, \
                                                         D, inv_bt, c, kl_beta, dmu, dlog_std, dvalue, daux, stats,  \
                                                         scratch)
    if (D <= 32) XB_PPGG(32);
    else XB_PPGG(64);
#undef XB_PPGG
    return xb_launch_status();
}

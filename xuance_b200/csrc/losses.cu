// K4 fused PPO-Clip loss forward+backward, K6 DQN TD target + loss forward+backward.
// Elementwise + row reductions over tiny rows (A <= 64 logits): one thread per sample, float4 loads when the
// row width allows, deterministic two-level reduction of the logged statistics.
#include "xb_common.cuh"

// =====================================================================================================
// K4  xb_ppo_loss_fwd_bwd
// =====================================================================================================
// Mirrors torch semantics of xuance/torch/learners/policy_gradient/ppo_learner.py:46-60:
//   Categorical(logits): logp_i = z_i - logsumexp(z);  entropy = -sum p_i*logp_i
//   torch.minimum backward: ties split the gradient in half; clamp backward passes inside [lo,hi] inclusive.
template <int A_MAX>
__global__ void __launch_bounds__(256, (A_MAX <= 4 ? 3 : 1)) ppo_loss_kernel(const float *__restrict__ logits,
                                                       const float *__restrict__ value,
                                                       const float *__restrict__ actions,
                                                       const float *__restrict__ old_logp,
                                                       const float *__restrict__ adv, const float *__restrict__ ret,
                                                       int64_t B, int A, float inv_bt, float clip, float vf_coef,
                                                       float ent_coef, int loss_kind, float *__restrict__ dlogits,
                                                       float *__restrict__ dvalue, float *__restrict__ stats,
                                                       double *__restrict__ scratch) {
    __shared__ double red[6 * 32];
    double acc[6] = {0, 0, 0, 0, 0, 0};  // a_loss, c_loss, entropy, v, clipped count, (unused)
    const float lo = 1.0f - clip, hi = 1.0f + clip;
    struct Row {
        float z[A_MAX];
        float v, act, ol, ad, r;
    };
    auto load_row = [&](int64_t b, Row &in) {
        const float *zr = logits + b * A;
        if (A_MAX == 4 && A == 4) {  // the BASELINE action count: one 16-byte load per row
            const float4 z4 = *reinterpret_cast<const float4 *>(zr);
            in.z[0] = z4.x, in.z[1] = z4.y, in.z[2] = z4.z, in.z[3] = z4.w;
        } else {
#pragma unroll
            for (int i = 0; i < A_MAX; ++i)
                if (i < A) in.z[i] = zr[i];
        }
        in.v = value[b], in.act = actions[b], in.ad = adv[b], in.r = ret[b];
        in.ol = (loss_kind == 0) ? old_logp[b] : 0.f;
    };
    auto compute_row = [&](int64_t b, const Row &in) {
        float m = -INFINITY;
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) m = fmaxf(m, in.z[i]);
        float se = 0.f;
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) se += expf(in.z[i] - m);
        const float lse = m + logf(se);
        const int a = (int)in.act;
        float ent = 0.f, logp_a = 0.f;
        float p[A_MAX], lp[A_MAX];
#pragma unroll
        for (int i = 0; i < A_MAX; ++i) {
            if (i < A) {
                lp[i] = in.z[i] - lse;
                p[i] = expf(lp[i]);
                ent -= p[i] * lp[i];
                if (i == a) logp_a = lp[i];
            }
        }
        const float ad = in.ad;
        float ratio = 1.f, smin, d_logp;
        if (loss_kind == 0) {  // PPO-Clip surrogate
            ratio = expf(logp_a - in.ol);
            const float rc = fminf(fmaxf(ratio, lo), hi);
            const float s1 = rc * ad, s2 = ad * ratio;
            smin = fminf(s1, s2);
            // d(-mean(min(s1,s2)))/d ratio
            float g1 = s1 < s2 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
            float g2 = s2 < s1 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
            const bool inside = ratio >= lo && ratio <= hi;
            const float d_ratio = -inv_bt * ad * ((inside ? g1 : 0.f) + g2);
            d_logp = d_ratio * ratio;  // d ratio / d logp = ratio
        } else {               // plain policy gradient: a_loss = -mean(w * logp)   (A2C: w = advantage, PG: w = return)
            smin = ad * logp_a;
            d_logp = -inv_bt * ad;
        }
        const float dent = -ent_coef * inv_bt;  // d loss / d entropy_b
        float *dz = dlogits + b * A;
        float gz[A_MAX];
#pragma unroll
        for (int i = 0; i < A_MAX; ++i) {
            if (i < A) {
                float g = d_logp * ((i == a ? 1.f : 0.f) - p[i]);  // d logp_a / d z_i
                g += dent * (-p[i] * (lp[i] + ent));               // d H / d z_i
                gz[i] = g;
            }
        }
        if (A_MAX == 4 && A == 4) {
            *reinterpret_cast<float4 *>(dz) = make_float4(gz[0], gz[1], gz[2], gz[3]);
        } else {
#pragma unroll
            for (int i = 0; i < A_MAX; ++i)
                if (i < A) dz[i] = gz[i];
        }
        const float dv = in.v - in.r;
        dvalue[b] = vf_coef * 2.f * dv * inv_bt;
        acc[0] += (double)(-smin);
        acc[1] += (double)dv * (double)dv;
        acc[2] += (double)ent;
        acc[3] += (double)in.v;
        acc[4] += (ratio < lo || ratio > hi) ? 1.0 : 0.0;
    };
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (A_MAX <= 4) {
        // two rows in flight per thread: the loads of the second row are issued before the (transcendental-heavy)
        // arithmetic of the first - the kernel is latency-bound on its global loads otherwise (ncu: long_scoreboard)
        for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += 2 * stride) {
            Row r0, r1;
            const bool two = b + stride < B;
            load_row(b, r0);
            if (two) load_row(b + stride, r1);
            compute_row(b, r0);
            if (two) compute_row(b + stride, r1);
        }
    } else {
        for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += stride) {
            Row r0;
            load_row(b, r0);
            compute_row(b, r0);
        }
    }
    grid_sum_finalize<6>(acc, scratch, red, [&](double(&t)[6]) {
        const double ib = (double)inv_bt;
        float a_loss = (float)(t[0] * ib), c_loss = (float)(t[1] * ib), e = (float)(t[2] * ib);
        stats[0] = a_loss;
        stats[1] = c_loss;
        stats[2] = e;
        stats[3] = (float)(t[3] * ib);
        stats[4] = (float)(t[4] * ib);
        stats[5] = a_loss - ent_coef * e + vf_coef * c_loss;
        stats[6] = 0.f;
        stats[7] = 0.f;
    });
}

extern "C" int xb_ppo_loss_fwd_bwd(const float *logits, const float *value, const float *actions,
                                   const float *old_logp, const float *adv, const float *ret, int64_t B, int A,
                                   int64_t B_total, float clip_range, float vf_coef, float ent_coef, int loss_kind,
                                   float *dlogits, float *dvalue, float *stats, double *scratch, void *stream) {
    if (!logits || !value || !actions || !adv || !ret || !dlogits || !dvalue || !stats || !scratch) return XB_EINVAL;
    if (loss_kind != 0 && loss_kind != 1) return XB_EINVAL;
    if (loss_kind == 0 && !old_logp) return XB_EINVAL;
    if (B <= 0 || B_total < B || A <= 0) return XB_EINVAL;
    if (A > 64) return XB_ERANGE;
    cudaStream_t s = (cudaStream_t)stream;
    int64_t want = (B + 255) / 256;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    const float inv_bt = 1.0f / (float)B_total;
    if (A == 4 && (!xb_aligned(logits, 16) || !xb_aligned(dlogits, 16))) return XB_EALIGN;
#define XB_PPO(AM)                                                                                                   \
    ppo_loss_kernel<AM><<<grid, 256, 0, s>>>(logits, value, actions, old_logp, adv, ret, B, A, inv_bt, clip_range,   \
                                              vf_coef, ent_coef, loss_kind, dlogits, dvalue, stats, scratch)
    if (A <= 4) XB_PPO(4);
    else if (A <= 8) XB_PPO(8);
    else if (A <= 18) XB_PPO(18);
    else if (A <= 32) XB_PPO(32);
    else XB_PPO(64);
#undef XB_PPO
    return xb_launch_status();
}

// =====================================================================================================
// K4G  xb_ppo_gauss_loss_fwd_bwd
// =====================================================================================================
// The same loss for a diagonal Gaussian policy: torch.distributions.Normal(mu, exp(log_std)) as the reference's
// DiagGaussianDistribution uses it (modules/distributions.py:165-197), log_prob and entropy summed over the D action
// components.  Per row, with z_j = (x_j - mu_j) / sigma_j:
//   logp = sum_j (-z_j^2/2 - log_std_j - log sqrt(2 pi))   (j in index order)   H = sum_j (1/2 + log(2 pi)/2 + log_std_j)
//   dmu_j = d_logp * z_j / sigma_j ;  d log_std_j (this row) = d_logp * (z_j^2 - 1) + dent
// log_std is shared by every row: each thread accumulates its rows' terms per column in float, each block adds its
// threads' sums in double in a fixed order and deposits one partial per column into ws[D][grid]; the last block to
// arrive adds the partials in block order.  No float atomics: dlog_std is bit-identical from launch to launch.
#define XB_LOG_SQRT_2PI 0.91893853320467274178f
template <int D_MAX>
__global__ void __launch_bounds__(256, 1) ppo_gauss_loss_kernel(
    const float *__restrict__ mu, const float *__restrict__ log_std, const float *__restrict__ value,
    const float *__restrict__ actions, const float *__restrict__ old_logp, const float *__restrict__ adv,
    const float *__restrict__ ret, int64_t B, int D, float inv_bt, float clip, float vf_coef, float ent_coef,
    int loss_kind, float *__restrict__ dmu, float *__restrict__ dlog_std, float *__restrict__ dvalue,
    float *__restrict__ stats, double *__restrict__ scratch, double *__restrict__ ws) {
    __shared__ double red[6 * 32];
    __shared__ double cred[D_MAX * 8];  // [column][warp] partials of the block (256 threads = 8 warps)
    __shared__ float s_ls[D_MAX], s_isig[D_MAX];
    for (int j = threadIdx.x; j < D; j += blockDim.x) {
        const float ls = log_std[j];
        s_ls[j] = ls;
        s_isig[j] = 1.f / expf(ls);
    }
    __syncthreads();
    float ent = 0.f;  // the same for every row
#pragma unroll
    for (int j = 0; j < D_MAX; ++j)
        if (j < D) ent += 0.5f + XB_LOG_SQRT_2PI + s_ls[j];
    double acc[6] = {0, 0, 0, 0, 0, 0};  // a_loss, c_loss, entropy, v, clipped count, (unused)
    double col_lo = 0.0, col_hi = 0.0;    // this warp's sums of the columns lane and lane + 32
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float lo = 1.0f - clip, hi = 1.0f + clip;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    // block-uniform trip count: every lane takes part in the column shuffles, rows past B contribute zero
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < B; base += stride) {
        const int64_t b = base + threadIdx.x;
        const bool active = b < B;
        const int64_t bb = active ? b : 0;
        const float *mr = mu + bb * D, *xr = actions + bb * D;
        float logp = 0.f;
#pragma unroll
        for (int j = 0; j < D_MAX; ++j) {
            if (j < D) {
                const float z = (xr[j] - mr[j]) * s_isig[j];
                logp += -0.5f * z * z - s_ls[j] - XB_LOG_SQRT_2PI;
            }
        }
        const float ad = adv[bb];
        float ratio = 1.f, smin, d_logp;
        if (loss_kind == 0) {  // PPO-Clip surrogate: K4's rules for ratio, clamp, min and their ties
            ratio = expf(logp - old_logp[bb]);
            const float rc = fminf(fmaxf(ratio, lo), hi);
            const float s1 = rc * ad, s2 = ad * ratio;
            smin = fminf(s1, s2);
            float g1 = s1 < s2 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
            float g2 = s2 < s1 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
            const bool inside = ratio >= lo && ratio <= hi;
            d_logp = -inv_bt * ad * ((inside ? g1 : 0.f) + g2) * ratio;
        } else {  // plain policy gradient (A2C / PG)
            smin = ad * logp;
            d_logp = -inv_bt * ad;
        }
        float *gr = dmu + b * D;
#pragma unroll
        for (int j = 0; j < D_MAX; ++j) {
            if (j < D) {
                const float z = (xr[j] - mr[j]) * s_isig[j];
                if (active) gr[j] = d_logp * z * s_isig[j];
                const double s = warp_sum_d(active ? (double)(d_logp * (z * z - 1.f)) : 0.0);
                if (j < 32) col_lo += (lane == j) ? s : 0.0;
                else col_hi += (lane == j - 32) ? s : 0.0;
            }
        }
        if (active) {
            const float v = value[b];
            const float dv = v - ret[b];
            dvalue[b] = vf_coef * 2.f * dv * inv_bt;
            acc[0] += (double)(-smin);
            acc[1] += (double)dv * (double)dv;
            acc[2] += (double)ent;
            acc[3] += (double)v;
            acc[4] += (ratio < lo || ratio > hi) ? 1.0 : 0.0;
        }
    }
    // column partials of this block: the 8 warps' sums in warp order
    if (lane < D) cred[lane * 8 + warp] = col_lo;
    if (lane + 32 < D) cred[(lane + 32) * 8 + warp] = col_hi;
    __syncthreads();
    if (threadIdx.x < D) {
        double s = 0.0;
        for (int w = 0; w < 8; ++w) s += cred[threadIdx.x * 8 + w];
        ws[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = s;
        __threadfence();
    }
    const bool last = grid_sum_finalize<6>(acc, scratch, red, [&](double(&t)[6]) {
        const double ib = (double)inv_bt;
        float a_loss = (float)(t[0] * ib), c_loss = (float)(t[1] * ib), e = (float)(t[2] * ib);
        stats[0] = a_loss;
        stats[1] = c_loss;
        stats[2] = e;
        stats[3] = (float)(t[3] * ib);
        stats[4] = (float)(t[4] * ib);
        stats[5] = a_loss - ent_coef * e + vf_coef * c_loss;
        stats[6] = 0.f;
        stats[7] = 0.f;
    });
    if (last && threadIdx.x < D) {
        const double *p = ws + (int64_t)threadIdx.x * gridDim.x;
        double s = 0.0;
        for (int k = 0; k < (int)gridDim.x; ++k) s += __ldcg(&p[k]);
        // the entropy term: d(-ent_coef * mean H)/d log_std_j = -ent_coef / B_total for each local row
        s += (double)B * (-(double)ent_coef * (double)inv_bt);
        dlog_std[threadIdx.x] = (float)s;
    }
}

extern "C" int64_t xb_ppo_gauss_ws_doubles(int64_t B, int D) {
    if (B <= 0 || D <= 0) return 0;
    const int64_t want = (B + 255) / 256;
    return (int64_t)D * (want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
}

extern "C" int xb_ppo_gauss_loss_fwd_bwd(const float *mu, const float *log_std, const float *value,
                                         const float *actions, const float *old_logp, const float *adv,
                                         const float *ret, int64_t B, int D, int64_t B_total, float clip_range,
                                         float vf_coef, float ent_coef, int loss_kind, float *dmu, float *dlog_std,
                                         float *dvalue, float *stats, double *scratch, double *ws,
                                         int64_t ws_doubles, void *stream) {
    if (!mu || !log_std || !value || !actions || !adv || !ret || !dmu || !dlog_std || !dvalue || !stats || !scratch ||
        !ws)
        return XB_EINVAL;
    if (loss_kind != 0 && loss_kind != 1) return XB_EINVAL;
    if (loss_kind == 0 && !old_logp) return XB_EINVAL;
    if (B <= 0 || B_total < B || D <= 0) return XB_EINVAL;
    if (D > 64) return XB_ERANGE;
    if (ws_doubles < xb_ppo_gauss_ws_doubles(B, D)) return XB_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    int64_t want = (B + 255) / 256;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    const float inv_bt = 1.0f / (float)B_total;
#define XB_PPOG(DM)                                                                                                  \
    ppo_gauss_loss_kernel<DM><<<grid, 256, 0, s>>>(mu, log_std, value, actions, old_logp, adv, ret, B, D, inv_bt,    \
                                                   clip_range, vf_coef, ent_coef, loss_kind, dmu, dlog_std, dvalue,  \
                                                   stats, scratch, ws)
    if (D <= 4) XB_PPOG(4);
    else if (D <= 8) XB_PPOG(8);
    else if (D <= 16) XB_PPOG(16);
    else if (D <= 32) XB_PPOG(32);
    else XB_PPOG(64);
#undef XB_PPOG
    return xb_launch_status();
}

// =====================================================================================================
// K6  xb_dqn_td_fwd_bwd
// =====================================================================================================
__global__ void __launch_bounds__(256) dqn_td_kernel(const float *__restrict__ q_eval, const float *__restrict__ q_next,
                                                     const float *__restrict__ q_sel,
                                                     const float *__restrict__ actions, const float *__restrict__ rew,
                                                     const float *__restrict__ term, int64_t B, int A, float inv_bt,
                                                     float gamma, float *__restrict__ dq, float *__restrict__ td,
                                                     float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[2 * 32];
    double acc[2] = {0, 0};
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const int a = (int)actions[b];
        const float *qe = q_eval + b * A, *qn = q_next + b * A;
        float mx = -INFINITY;
        if (q_sel) {  // double-Q: evaluate the target net at the eval net's greedy action (ddqn_learner.py:39-44)
            const float *qs = q_sel + b * A;
            int best = 0;
            float bv = qs[0];
            for (int i = 1; i < A; ++i)
                if (qs[i] > bv) {  // first maximal index, as torch.argmax
                    bv = qs[i];
                    best = i;
                }
            mx = qn[best];
        } else {
            for (int i = 0; i < A; ++i) mx = fmaxf(mx, qn[i]);
        }
        const float pred = qe[a];
        // targetQ = rew + gamma*(1-ter)*max  evaluated left to right as torch does: (gamma*(1-ter))*max
        const float y = __fadd_rn(rew[b], __fmul_rn(__fmul_rn(gamma, __fsub_rn(1.f, term[b])), mx));
        const float e = __fsub_rn(y, pred);  // td_error = targetQ - predictQ
        td[b] = e;
        float *g = dq + b * A;
        const float ga = -2.f * e * inv_bt;  // d mean((pred-y)^2) / d pred
        for (int i = 0; i < A; ++i) g[i] = (i == a) ? ga : 0.f;
        acc[0] += (double)e * (double)e;
        acc[1] += (double)pred;
    }
    grid_sum_finalize<2>(acc, scratch, red, [&](double(&t)[2]) {
        stats[0] = (float)(t[0] * (double)inv_bt);
        stats[1] = (float)(t[1] * (double)inv_bt);
        stats[2] = 0.f;
        stats[3] = 0.f;
    });
}

extern "C" int xb_dqn_td_fwd_bwd(const float *q_eval, const float *q_next, const float *q_sel, const float *actions,
                                 const float *rew,
                                 const float *term, int64_t B, int A, int64_t B_total, float gamma, float *dq,
                                 float *td, float *stats, double *scratch, void *stream) {
    if (!q_eval || !q_next || !actions || !rew || !term || !dq || !td || !stats || !scratch) return XB_EINVAL;
    if (B <= 0 || B_total < B || A <= 0) return XB_EINVAL;
    int64_t want = (B + 255) / 256;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    dqn_td_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(q_eval, q_next, q_sel, actions, rew, term, B, A,
                                                          1.0f / (float)B_total, gamma, dq, td, stats, scratch);
    return xb_launch_status();
}

// =====================================================================================================
// K4M  xb_mappo_prepare / xb_value_norm_update / xb_mappo_loss_fwd_bwd
// =====================================================================================================
// MAPPO_Learner.update (mappo_learner.py:55-113) for one parameter-sharing group of a feed-forward actor and critic.
// prepare: block[0..2] = (sum mask, sum ret, sum ret^2) over the local rows in float64 (deterministic grid reduction);
// the learner SUM-all-reduces the block when the minibatch is sharded.
__global__ void __launch_bounds__(256) mappo_prepare_kernel(const float *__restrict__ mask, const float *__restrict__ ret,
                                                            int64_t R, double *__restrict__ block,
                                                            double *__restrict__ scratch) {
    __shared__ double red[3 * 32];
    double acc[3] = {0, 0, 0};
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < R; b += (int64_t)gridDim.x * blockDim.x) {
        const double r = (double)ret[b];
        acc[0] += (double)mask[b];
        acc[1] += r;
        acc[2] += r * r;
    }
    grid_sum_finalize<3>(acc, scratch, red, [&](double(&t)[3]) {
        block[0] = t[0];
        block[1] = t[1];
        block[2] = t[2];
        block[3] = 0.0;
    });
}

extern "C" int xb_mappo_prepare(const float *mask, const float *ret, int64_t R, double *block, double *scratch,
                                void *stream) {
    if (!mask || !ret || !block || !scratch || R <= 0) return XB_EINVAL;
    const int64_t want = (R + 255) / 256;
    const int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    mappo_prepare_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(mask, ret, R, block, scratch);
    return xb_launch_status();
}

// ValueNorm.running_mean_var (value_norm.py:29-33) in float32, in torch's operation order.
__device__ __forceinline__ void value_norm_mean_std(float rm, float rmsq, float dt, float &mean, float &stdv) {
    const float d = fmaxf(dt, 1e-5f);
    mean = __fdiv_rn(rm, d);
    const float msq = __fdiv_rn(rmsq, d);
    const float var = fmaxf(__fsub_rn(msq, __fmul_rn(mean, mean)), 1e-2f);
    stdv = __fsqrt_rn(var);
}

// ValueNorm.update (value_norm.py:35-52, per_element_update=False) on the batch moments of the prepared block, then
// (mean, std) of the updated state into mean_std[2].
__global__ void value_norm_update_kernel(float *rm, float *rmsq, float *dt, const double *block, int64_t R_total,
                                         float w, float omw, float *mean_std) {
    const float bm = (float)(block[1] / (double)R_total);
    const float bsq = (float)(block[2] / (double)R_total);
    const float m = __fadd_rn(__fmul_rn(rm[0], w), __fmul_rn(bm, omw));
    const float msq = __fadd_rn(__fmul_rn(rmsq[0], w), __fmul_rn(bsq, omw));
    const float d = __fadd_rn(__fmul_rn(dt[0], w), omw);
    rm[0] = m, rmsq[0] = msq, dt[0] = d;
    float mean, stdv;
    value_norm_mean_std(m, msq, d, mean, stdv);
    mean_std[0] = mean;
    mean_std[1] = stdv;
}

extern "C" int xb_value_norm_update(float *running_mean, float *running_mean_sq, float *debiasing_term,
                                    const double *block, int64_t R_total, double beta, float *mean_std, void *stream) {
    if (!running_mean || !running_mean_sq || !debiasing_term || !block || !mean_std || R_total <= 0) return XB_EINVAL;
    if (!(beta > 0.0 && beta < 1.0)) return XB_EINVAL;
    value_norm_update_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(running_mean, running_mean_sq, debiasing_term, block,
                                                                R_total, (float)beta, (float)(1.0 - beta), mean_std);
    return xb_launch_status();
}

template <int A_MAX>
__global__ void __launch_bounds__(256, 1) mappo_loss_kernel(
    const float *__restrict__ logits, const uint8_t *__restrict__ avail, int avail_ld,
    const float *__restrict__ actions, const float *__restrict__ old_logp, const float *__restrict__ adv,
    const float *__restrict__ value, const float *__restrict__ old_value, const float *__restrict__ ret,
    const float *__restrict__ mask, const float *__restrict__ vn, const double *__restrict__ prep, int64_t R, int A,
    int64_t R_total, float clip, float vclip, float hdelta, float vf_coef, float ent_coef,
    float *__restrict__ dlogits, float *__restrict__ dvalue, float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[4 * 32];
    double acc[4] = {0, 0, 0, 0};  // sum mask*(-min surrogate), mask*critic loss, mask*entropy, value
    const double msum = prep[0];
    // the reference divides by mask.sum(): with a global sum of 0 every weight is 0/0 = NaN, as there
    const float inv_ms = (float)(1.0 / msum);
    const float lo = 1.0f - clip, hi = 1.0f + clip;
    float vmean = 0.f, vstd = 1.f;
    if (vn) vmean = vn[0], vstd = vn[1];
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < R; b += (int64_t)gridDim.x * blockDim.x) {
        const float *zr = logits + b * A;
        const uint8_t *av = avail ? avail + b * avail_ld : nullptr;
        float z[A_MAX];
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) z[i] = (av && !av[i]) ? -1e10f : zr[i];  // actor_head.py:40 (in place: no gradient there)
        float m = -INFINITY;
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) m = fmaxf(m, z[i]);
        float se = 0.f;
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) se += expf(z[i] - m);
        const float lse = m + logf(se);
        const int a = (int)actions[b];
        float ent = 0.f, logp_a = 0.f;
#pragma unroll
        for (int i = 0; i < A_MAX; ++i) {
            if (i < A) {
                const float lp = z[i] - lse;
                ent -= expf(lp) * lp;
                if (i == a) logp_a = lp;
            }
        }
        const float mk = mask[b], w = mk * inv_ms;
        const float ad = adv[b];
        // policy: -(min(ratio*adv, clip(ratio)*adv) * mask).sum() / mask.sum()
        const float ratio = expf(logp_a - old_logp[b]);
        const float rc = fminf(fmaxf(ratio, lo), hi);
        const float s1 = ratio * ad, s2 = rc * ad;
        const float smin = fminf(s1, s2);
        const float g1 = s1 < s2 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
        const float g2 = s2 < s1 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
        const bool inside = ratio >= lo && ratio <= hi;  // clamp backward passes the gradient on the boundary
        const float d_logp = -w * ad * (g1 + (inside ? g2 : 0.f)) * ratio;
        const float dent = -ent_coef * w;
        float *dz = dlogits + b * A;
#pragma unroll
        for (int i = 0; i < A_MAX; ++i) {
            if (i < A) {
                const float lp = z[i] - lse, p = expf(lp);
                float g = d_logp * ((i == a ? 1.f : 0.f) - p) + dent * (-p * (lp + ent));
                dz[i] = (av && !av[i]) ? 0.f : g;
            }
        }
        // critic: value clipping, value normalisation of the target, Huber or squared error, torch.max of the two
        const float vp = value[b];
        const float tgt = vn ? __fdiv_rn(__fsub_rn(ret[b], vmean), vstd) : ret[b];
        float l1, gv1, lc, dlc;
        value_loss(__fsub_rn(vp, tgt), hdelta, l1, gv1);
        if (vclip > 0.f) {
            const float vo = old_value[b];
            const float dd = __fsub_rn(vp, vo);
            const float vc = __fadd_rn(vo, fminf(fmaxf(dd, -vclip), vclip));
            const bool pass = dd >= -vclip && dd <= vclip;
            float l2, gv2;
            value_loss(__fsub_rn(vc, tgt), hdelta, l2, gv2);
            lc = fmaxf(l1, l2);
            const float h1 = l1 > l2 ? 1.f : (l1 == l2 ? 0.5f : 0.f);
            const float h2 = l2 > l1 ? 1.f : (l1 == l2 ? 0.5f : 0.f);
            dlc = h1 * gv1 + (pass ? h2 * gv2 : 0.f);
        } else {
            lc = l1;
            dlc = gv1;
        }
        dvalue[b] = vf_coef * w * dlc;
        acc[0] += (double)(-smin) * (double)mk;
        acc[1] += (double)lc * (double)mk;
        acc[2] += (double)ent * (double)mk;
        acc[3] += (double)vp;
    }
    grid_sum_finalize<4>(acc, scratch, red, [&](double(&t)[4]) {
        const double im = 1.0 / msum;
        const float a_loss = (float)(t[0] * im), c_loss = (float)(t[1] * im), e = (float)(t[2] * im);
        stats[0] = a_loss;
        stats[1] = c_loss;
        stats[2] = e;
        stats[3] = (float)(t[3] / (double)R_total);
        stats[4] = a_loss + vf_coef * c_loss - ent_coef * e;
        stats[5] = 0.f;
        stats[6] = 0.f;
        stats[7] = 0.f;
    });
}

extern "C" int xb_mappo_loss_fwd_bwd(const float *logits, const uint8_t *avail, int avail_ld, const float *actions,
                                     const float *old_logp, const float *adv, const float *value,
                                     const float *old_value, const float *ret, const float *mask, const float *vn,
                                     const double *prep, int64_t R, int A, int64_t R_total, float clip_range,
                                     float value_clip_range, float huber_delta, float vf_coef, float ent_coef,
                                     float *dlogits, float *dvalue, float *stats, double *scratch, void *stream) {
    if (!logits || !actions || !old_logp || !adv || !value || !ret || !mask || !prep || !dlogits || !dvalue ||
        !stats || !scratch)
        return XB_EINVAL;
    if (value_clip_range > 0.f && !old_value) return XB_EINVAL;
    if (R <= 0 || R_total < R || A <= 0) return XB_EINVAL;
    if (avail && avail_ld < A) return XB_EINVAL;
    if (A > 64) return XB_ERANGE;
    const int64_t want = (R + 255) / 256;
    const int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    cudaStream_t s = (cudaStream_t)stream;
#define XB_MAPPO(AM)                                                                                                 \
    mappo_loss_kernel<AM><<<grid, 256, 0, s>>>(logits, avail, avail_ld, actions, old_logp, adv, value, old_value,   \
                                               ret, mask, vn, prep, R, A, R_total, clip_range, value_clip_range,     \
                                               huber_delta, vf_coef, ent_coef, dlogits, dvalue, stats, scratch)
    if (A <= 4) XB_MAPPO(4);
    else if (A <= 8) XB_MAPPO(8);
    else if (A <= 18) XB_MAPPO(18);
    else if (A <= 32) XB_MAPPO(32);
    else XB_MAPPO(64);
#undef XB_MAPPO
    return xb_launch_status();
}

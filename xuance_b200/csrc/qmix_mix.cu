// K6 QMIX: (a) action-value selection over the padded episode batch, (b) the per-row monotonic mixing network
// (abs / batched [1 x n]x[n x H] and [1 x H]x[H x 1] contractions / ELU) forward and backward, (c) masked TD loss.
// One warp per (episode, step) row: lane j owns hidden unit j (H <= 32 per pass), the n agent utilities are
// broadcast, the two contractions are warp-shuffle reductions.  The hypernetwork linear layers that produce
// w1/b1/w2/b2 from the global state are plain GEMMs and stay in cuBLAS (include/xb200.h, K6).
#include "xb_common.cuh"

// =====================================================================================================
// (a) selection:  q_eval_taken[b*T+t, i] = Q[b,i,t,a_{b,i,t}] * mask ;  q_next_taken = Q'[b,i,t+1, argmax/max] * mask
// =====================================================================================================
// Layouts: q_all, q_tgt [B, n, T+1, A]; actions, agent_mask [B, n, T] (float32); filled [B, T] (float32).
// avail (nullable): uint8 [B, n, T+1, avail_ld], non-zero = the action is available at that step.  With it, the double-Q
// arg-max runs over the eval values with unavailable actions at -1e10 and the target values of unavailable actions are
// -1e10 before the gather / max - iql_learner.py:60-81 with the time axis sliced ([:, :, 1:], the evidently intended
// indexing; the reference slices the agent axis and crashes for use_rnn, DESIGN.md section 4).
// One thread per (b, i, t).  Also accumulates sum(filled) (needed by the masked loss) deterministically.
__global__ void __launch_bounds__(256) qmix_select_fwd_kernel(const float *__restrict__ q_all,
                                                              const float *__restrict__ q_tgt,
                                                              const float *__restrict__ actions,
                                                              const float *__restrict__ agent_mask,
                                                              const float *__restrict__ filled,
                                                              const uint8_t *__restrict__ avail, int avail_ld, int B,
                                                              int n, int T, int A, int double_q,
                                                              float *__restrict__ q_eval_taken,
                                                              float *__restrict__ q_next_taken,
                                                              float *__restrict__ filled_sum,
                                                              double *__restrict__ scratch) {
    __shared__ double red[32];
    double acc[1] = {0.0};
    const int64_t total = (int64_t)B * n * T;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int t = (int)(e % T);
        const int i = (int)((e / T) % n);
        const int b = (int)(e / ((int64_t)T * n));
        const float m = agent_mask[e] * filled[(int64_t)b * T + t];
        const float *qe = q_all + (((int64_t)b * n + i) * (T + 1) + t) * A;
        const float *qe1 = qe + A;  // step t+1 of the eval network (double-Q argmax)
        const float *qt1 = q_tgt + (((int64_t)b * n + i) * (T + 1) + t + 1) * A;
        const int a = (int)actions[e];
        const uint8_t *av1 = avail ? avail + (((int64_t)b * n + i) * (T + 1) + t + 1) * avail_ld : nullptr;
        const float NEG = -1e10f;
        float nxt;
        if (double_q) {
            int best = 0;
            float bv = (av1 && !av1[0]) ? NEG : qe1[0];
            for (int k = 1; k < A; ++k) {
                const float v = (av1 && !av1[k]) ? NEG : qe1[k];
                if (v > bv) {  // torch.argmax: first maximal index
                    bv = v;
                    best = k;
                }
            }
            nxt = (av1 && !av1[best]) ? NEG : qt1[best];
        } else {
            nxt = (av1 && !av1[0]) ? NEG : qt1[0];
            for (int k = 1; k < A; ++k) nxt = fmaxf(nxt, (av1 && !av1[k]) ? NEG : qt1[k]);
        }
        const int64_t row = (int64_t)b * T + t;
        q_eval_taken[row * n + i] = qe[a] * m;
        q_next_taken[row * n + i] = nxt * m;
        if (i == 0) acc[0] += (double)filled[row];
    }
    grid_sum_finalize<1>(acc, scratch, red, [&](double(&tot)[1]) { filled_sum[0] = (float)tot[0]; });
}

// backward of the eval selection: dq_all[b,i,t,a] = d_taken[row,i] * mask  (dq_all pre-zeroed by the caller)
__global__ void __launch_bounds__(256) qmix_select_bwd_kernel(const float *__restrict__ d_taken,
                                                              const float *__restrict__ actions,
                                                              const float *__restrict__ agent_mask,
                                                              const float *__restrict__ filled, int B, int n, int T,
                                                              int A, float *__restrict__ dq_all) {
    const int64_t total = (int64_t)B * n * T;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int t = (int)(e % T);
        const int i = (int)((e / T) % n);
        const int b = (int)(e / ((int64_t)T * n));
        const float m = agent_mask[e] * filled[(int64_t)b * T + t];
        const int a = (int)actions[e];
        dq_all[(((int64_t)b * n + i) * (T + 1) + t) * A + a] = d_taken[((int64_t)b * T + t) * n + i] * m;
    }
}

extern "C" int xb_qmix_select_fwd(const float *q_all, const float *q_tgt, const float *actions,
                                  const float *agent_mask, const float *filled, const uint8_t *avail, int avail_ld,
                                  int B, int n, int T, int A, int double_q, float *q_eval_taken, float *q_next_taken,
                                  float *filled_sum, double *scratch, void *stream) {
    if (!q_all || !q_tgt || !actions || !agent_mask || !filled || !q_eval_taken || !q_next_taken || !filled_sum ||
        !scratch)
        return XB_EINVAL;
    if (B <= 0 || n <= 0 || T <= 0 || A <= 0 || (avail && avail_ld < A)) return XB_EINVAL;
    int64_t total = (int64_t)B * n * T, want = (total + 255) / 256;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    qmix_select_fwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(q_all, q_tgt, actions, agent_mask, filled, avail,
                                                                   avail_ld, B, n, T, A, double_q, q_eval_taken,
                                                                   q_next_taken, filled_sum, scratch);
    return xb_launch_status();
}

extern "C" int xb_qmix_select_bwd(const float *d_taken, const float *actions, const float *agent_mask,
                                  const float *filled, int B, int n, int T, int A, float *dq_all, void *stream) {
    if (!d_taken || !actions || !agent_mask || !filled || !dq_all) return XB_EINVAL;
    if (B <= 0 || n <= 0 || T <= 0 || A <= 0) return XB_EINVAL;
    int64_t total = (int64_t)B * n * T, want = (total + 255) / 256;
    int64_t cap = (int64_t)xb_sm_count() * 8;
    qmix_select_bwd_kernel<<<(int)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(d_taken, actions, agent_mask,
                                                                                           filled, B, n, T, A, dq_all);
    return xb_launch_status();
}

// =====================================================================================================
// (b) mixing network epilogue (xuance/torch/rl_models/heads/q_mix_head.py:66-95)
//     hidden = elu(q . |w1| + b1) ; q_tot = hidden . |w2| + b2          per row
// =====================================================================================================
// w1_raw [R, n*H] (row-major [n][H] per row), b1 [R, H], w2_raw [R, H], b2 [R], q [R, n].  Warp per row.
__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : (expf(x) - 1.f); }

__global__ void __launch_bounds__(256) qmix_mix_fwd_kernel(const float *__restrict__ q, const float *__restrict__ w1,
                                                           const float *__restrict__ b1, const float *__restrict__ w2,
                                                           const float *__restrict__ b2, int64_t R, int n, int H,
                                                           float *__restrict__ q_tot) {
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp0; r < R; r += nwarps) {
        const float *w1r = w1 + r * (int64_t)n * H;
        float part = 0.f;
        for (int j = lane; j < H; j += 32) {
            float pre = b1[r * H + j];
            for (int i = 0; i < n; ++i) pre += q[r * n + i] * fabsf(w1r[i * H + j]);
            part += elu1(pre) * fabsf(w2[r * H + j]);
        }
        part = warp_sum_f(part);
        if (lane == 0) q_tot[r] = part + b2[r];
    }
}

__global__ void __launch_bounds__(256) qmix_mix_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ q,
                                                           const float *__restrict__ w1, const float *__restrict__ b1,
                                                           const float *__restrict__ w2, int64_t R, int n, int H,
                                                           float *__restrict__ dq, float *__restrict__ dw1,
                                                           float *__restrict__ db1, float *__restrict__ dw2) {
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp0; r < R; r += nwarps) {
        const float g = dy[r];
        const float *w1r = w1 + r * (int64_t)n * H;
        float *dw1r = dw1 + r * (int64_t)n * H;
        float dq_acc[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) dq_acc[i] = 0.f;
        for (int j = lane; j < H; j += 32) {
            float pre = b1[r * H + j];
            for (int i = 0; i < n; ++i) pre += q[r * n + i] * fabsf(w1r[i * H + j]);
            const float h = elu1(pre);
            const float w2v = w2[r * H + j];
            const float sgn2 = (w2v > 0.f) - (w2v < 0.f);
            dw2[r * H + j] = g * h * sgn2;
            const float dpre = g * fabsf(w2v) * (pre > 0.f ? 1.f : (h + 1.f));  // elu' = exp(pre) = h + 1
            db1[r * H + j] = dpre;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                if (i < n) {
                    const float wv = w1r[i * H + j];
                    const float sgn = (wv > 0.f) - (wv < 0.f);
                    dw1r[i * H + j] = dpre * q[r * n + i] * sgn;
                    dq_acc[i] += dpre * fabsf(wv);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            if (i < n) {
                float s = warp_sum_f(dq_acc[i]);
                if (lane == 0) dq[r * n + i] = s;
            }
        }
    }
}

// ---- H == 32 fast path: 8 lanes per row (4 rows per warp), each lane owns 4 hidden units through 16-byte loads
__device__ __forceinline__ float4 abs4(float4 v) { return make_float4(fabsf(v.x), fabsf(v.y), fabsf(v.z), fabsf(v.w)); }
__device__ __forceinline__ float sum8(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}
__device__ __forceinline__ float sgnf(float v) { return (float)((v > 0.f) - (v < 0.f)); }

template <int N_MAX>
__global__ void __launch_bounds__(256) qmix_mix_fwd_h32_kernel(const float *__restrict__ q, const float *__restrict__ w1,
                                                               const float *__restrict__ b1, const float *__restrict__ w2,
                                                               const float *__restrict__ b2, int64_t R, int n,
                                                               float *__restrict__ q_tot) {
    const int sub = threadIdx.x & 7;
    const int64_t grp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const int64_t ngrp = ((int64_t)gridDim.x * blockDim.x) >> 3;
    const int64_t Rp = (R + 3) & ~(int64_t)3;  // whole warps stay converged (4 rows per warp)
    for (int64_t r = grp0; r < Rp; r += ngrp) {
        const bool live = r < R;
        const int64_t rr = live ? r : R - 1;
        float4 pre = *reinterpret_cast<const float4 *>(b1 + rr * 32 + sub * 4);
#pragma unroll
        for (int i = 0; i < N_MAX; ++i) {
            if (i < n) {
                const float qi = q[rr * n + i];
                const float4 w = abs4(*reinterpret_cast<const float4 *>(w1 + (rr * n + i) * 32 + sub * 4));
                pre.x += qi * w.x, pre.y += qi * w.y, pre.z += qi * w.z, pre.w += qi * w.w;
            }
        }
        const float4 w2v = abs4(*reinterpret_cast<const float4 *>(w2 + rr * 32 + sub * 4));
        float part = elu1(pre.x) * w2v.x + elu1(pre.y) * w2v.y + elu1(pre.z) * w2v.z + elu1(pre.w) * w2v.w;
        part = sum8(part);
        if (live && sub == 0) q_tot[r] = part + b2[r];
    }
}

template <int N_MAX>
__global__ void __launch_bounds__(256) qmix_mix_bwd_h32_kernel(const float *__restrict__ dy, const float *__restrict__ q,
                                                               const float *__restrict__ w1, const float *__restrict__ b1,
                                                               const float *__restrict__ w2, int64_t R, int n,
                                                               float *__restrict__ dq, float *__restrict__ dw1,
                                                               float *__restrict__ db1, float *__restrict__ dw2) {
    const int sub = threadIdx.x & 7;
    const int64_t grp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const int64_t ngrp = ((int64_t)gridDim.x * blockDim.x) >> 3;
    const int64_t Rp = (R + 3) & ~(int64_t)3;
    for (int64_t r = grp0; r < Rp; r += ngrp) {
        const bool live = r < R;
        const int64_t rr = live ? r : R - 1;
        const float g = dy[rr];
        float qv[N_MAX];
        float4 wv[N_MAX];
        float4 pre = *reinterpret_cast<const float4 *>(b1 + rr * 32 + sub * 4);
#pragma unroll
        for (int i = 0; i < N_MAX; ++i) {
            if (i < n) {
                qv[i] = q[rr * n + i];
                wv[i] = *reinterpret_cast<const float4 *>(w1 + (rr * n + i) * 32 + sub * 4);
                pre.x += qv[i] * fabsf(wv[i].x), pre.y += qv[i] * fabsf(wv[i].y);
                pre.z += qv[i] * fabsf(wv[i].z), pre.w += qv[i] * fabsf(wv[i].w);
            }
        }
        const float4 w2v = *reinterpret_cast<const float4 *>(w2 + rr * 32 + sub * 4);
        const float4 h = make_float4(elu1(pre.x), elu1(pre.y), elu1(pre.z), elu1(pre.w));
        const float4 dpre = make_float4(g * fabsf(w2v.x) * (pre.x > 0.f ? 1.f : h.x + 1.f),
                                        g * fabsf(w2v.y) * (pre.y > 0.f ? 1.f : h.y + 1.f),
                                        g * fabsf(w2v.z) * (pre.z > 0.f ? 1.f : h.z + 1.f),
                                        g * fabsf(w2v.w) * (pre.w > 0.f ? 1.f : h.w + 1.f));
        if (live) {
            *reinterpret_cast<float4 *>(dw2 + r * 32 + sub * 4) =
                make_float4(g * h.x * sgnf(w2v.x), g * h.y * sgnf(w2v.y), g * h.z * sgnf(w2v.z), g * h.w * sgnf(w2v.w));
            *reinterpret_cast<float4 *>(db1 + r * 32 + sub * 4) = dpre;
        }
#pragma unroll
        for (int i = 0; i < N_MAX; ++i) {
            if (i < n) {
                if (live)
                    *reinterpret_cast<float4 *>(dw1 + (r * n + i) * 32 + sub * 4) =
                        make_float4(dpre.x * qv[i] * sgnf(wv[i].x), dpre.y * qv[i] * sgnf(wv[i].y),
                                    dpre.z * qv[i] * sgnf(wv[i].z), dpre.w * qv[i] * sgnf(wv[i].w));
                float s = dpre.x * fabsf(wv[i].x) + dpre.y * fabsf(wv[i].y) + dpre.z * fabsf(wv[i].z) +
                          dpre.w * fabsf(wv[i].w);
                s = sum8(s);
                if (live && sub == 0) dq[r * n + i] = s;
            }
        }
    }
}

static inline bool mix_fast_ok(int H, int n, const void *a, const void *b, const void *c, const void *d = nullptr,
                               const void *e = nullptr, const void *f = nullptr) {
    return H == 32 && n <= 8 && xb_aligned(a, 16) && xb_aligned(b, 16) && xb_aligned(c, 16) &&
           (!d || xb_aligned(d, 16)) && (!e || xb_aligned(e, 16)) && (!f || xb_aligned(f, 16));
}

extern "C" int xb_qmix_mix_fwd(const float *q, const float *w1_raw, const float *b1, const float *w2_raw,
                               const float *b2, int64_t R, int n, int H, float *q_tot, void *stream) {
    if (!q || !w1_raw || !b1 || !w2_raw || !b2 || !q_tot || R <= 0 || n <= 0 || H <= 0) return XB_EINVAL;
    if (n > 16) return XB_ERANGE;
    int64_t cap = (int64_t)xb_sm_count() * 8;
    if (mix_fast_ok(H, n, w1_raw, b1, w2_raw)) {
        int64_t want = (R * 8 + 255) / 256;
        qmix_mix_fwd_h32_kernel<8><<<(int)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(q, w1_raw, b1, w2_raw,
                                                                                                  b2, R, n, q_tot);
        return xb_launch_status();
    }
    int64_t want = (R * 32 + 255) / 256;
    qmix_mix_fwd_kernel<<<(int)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(q, w1_raw, b1, w2_raw, b2, R, n,
                                                                                        H, q_tot);
    return xb_launch_status();
}

extern "C" int xb_qmix_mix_bwd(const float *dq_tot, const float *q, const float *w1_raw, const float *b1,
                               const float *w2_raw, int64_t R, int n, int H, float *dq, float *dw1_raw, float *db1,
                               float *dw2_raw, void *stream) {
    if (!dq_tot || !q || !w1_raw || !b1 || !w2_raw || !dq || !dw1_raw || !db1 || !dw2_raw) return XB_EINVAL;
    if (R <= 0 || n <= 0 || H <= 0) return XB_EINVAL;
    if (n > 16) return XB_ERANGE;
    int64_t cap = (int64_t)xb_sm_count() * 8;
    if (mix_fast_ok(H, n, w1_raw, b1, w2_raw, dw1_raw, db1, dw2_raw)) {
        int64_t want = (R * 8 + 255) / 256;
        qmix_mix_bwd_h32_kernel<8><<<(int)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(
            dq_tot, q, w1_raw, b1, w2_raw, R, n, dq, dw1_raw, db1, dw2_raw);
        return xb_launch_status();
    }
    int64_t want = (R * 32 + 255) / 256;
    qmix_mix_bwd_kernel<<<(int)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(dq_tot, q, w1_raw, b1, w2_raw, R,
                                                                                        n, H, dq, dw1_raw, db1, dw2_raw);
    return xb_launch_status();
}

// =====================================================================================================
// (c) masked TD loss (qmix_learner.py:34-35, 76-84): team reward = mean over agents, team terminal = all agents,
//     y = r + (1-d)*gamma*Qtot' ; td = (Qtot - y)*filled ; loss = sum(td^2)/sum(filled) ; dQtot = 2*td*filled/sum(filled)
// Both denominators are global (filled_sum all-reduced, rows_total = B*T over all ranks), so a rank-local shard writes
// its share of the global sums, like K4/K6/K8.
// =====================================================================================================
__global__ void __launch_bounds__(256) qmix_td_kernel(const float *__restrict__ q_tot, const float *__restrict__ q_tot_next,
                                                      const float *__restrict__ rewards,
                                                      const float *__restrict__ terminals,
                                                      const float *__restrict__ filled,
                                                      const float *__restrict__ filled_sum, int B, int n, int T,
                                                      float gamma, int64_t rows_total, float *__restrict__ dq_tot,
                                                      float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[2 * 32];
    double acc[2] = {0, 0};
    const float fs = filled_sum[0];
    const int64_t R = (int64_t)B * T;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < R; row += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(row / T), t = (int)(row % T);
        float rs = 0.f;
        bool all_term = true;
        for (int i = 0; i < n; ++i) {
            const int64_t e = ((int64_t)b * n + i) * T + t;
            rs += rewards[e];
            all_term = all_term && (terminals[e] != 0.f);
        }
        const float r_tot = rs / (float)n;
        const float d_tot = all_term ? 1.f : 0.f;
        const float y = r_tot + (1.f - d_tot) * gamma * q_tot_next[row];
        const float f = filled[row];
        const float td = (q_tot[row] - y) * f;
        dq_tot[row] = 2.f * td * f / fs;
        acc[0] += (double)td * td;
        acc[1] += (double)q_tot[row];
    }
    grid_sum_finalize<2>(acc, scratch, red, [&](double(&tsum)[2]) {
        stats[0] = (float)(tsum[0] / (double)fs);            // loss_Q
        stats[1] = (float)(tsum[1] / (double)rows_total);    // predictQ = mean(q_tot_eval)
    });
}

extern "C" int xb_qmix_td(const float *q_tot, const float *q_tot_next, const float *rewards, const float *terminals,
                          const float *filled, const float *filled_sum, int B, int n, int T, float gamma,
                          int64_t rows_total, float *dq_tot, float *stats, double *scratch, void *stream) {
    if (!q_tot || !q_tot_next || !rewards || !terminals || !filled || !filled_sum || !dq_tot || !stats || !scratch)
        return XB_EINVAL;
    if (B <= 0 || n <= 0 || T <= 0) return XB_EINVAL;
    int64_t R = (int64_t)B * T, want = (R + 255) / 256;
    if (rows_total < R) return XB_EINVAL;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    qmix_td_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(q_tot, q_tot_next, rewards, terminals, filled, filled_sum, B, n,
                                                           T, gamma, rows_total, dq_tot, stats, scratch);
    return xb_launch_status();
}

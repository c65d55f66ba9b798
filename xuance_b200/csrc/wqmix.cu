// K9W Weighted QMIX (OW-QMIX / CW-QMIX, wqmix_learner.py:27-227): (a) the three per-agent selections of
// _forward_transitions plus the greedy indices, the CW agreement flag and sum(filled) in one pass, (b) the scatter of
// both differentiable selections back into the agent-network outputs, (c) the weighted masked TD loss of the QMIX mixer
// together with the unweighted loss of the feed-forward (central) mixer.  The mixers themselves are the K9 mix kernels
// (QMIX hypernetwork mixer) and cuBLAS (QMIX_FF_Mixer); see include/xb200.h, K9W.
#include "xb_common.cuh"

// First maximal index of q[0..A) with unavailable actions counted as -1e10 (value_factorization.py:86-91; torch.argmax
// keeps the first of equal values).  av == NULL: every action is available.
__device__ __forceinline__ int wq_argmax(const float *__restrict__ q, const uint8_t *__restrict__ av, int A) {
    const float NEG = -1e10f;
    int best = 0;
    float bv = (av && !av[0]) ? NEG : q[0];
    for (int k = 1; k < A; ++k) {
        const float v = (av && !av[k]) ? NEG : q[k];
        if (v > bv) {
            bv = v;
            best = k;
        }
    }
    return best;
}

// =====================================================================================================
// (a) selection.  One thread per (episode, step) row; it walks the n agents so the CW flag needs no cross-thread step.
//   g_t      = argmax_masked q_all[b,i,t]                          (the eval networks' greedy action at t)
//   a_next   = double_q ? argmax_masked q_all[b,i,t+1] : argmax q_tgt[b,i,t+1]  (the latter unmasked, as the reference's
//              use_rnn branch never applies the -1e10 mask to q_next)
//   q_eval_taken[row,i] = q_all[b,i,t,a_t] * m ; q_cent_taken[row,i] = q_cent[b,i,t,g_t] * m ;
//   q_next_cent[row,i]  = q_cent_tgt[b,i,t+1,a_next] * m ;           m = agent_mask[b,i,t] * filled[b,t]
//   agree[row] = all_i (g_t == a_t && m != 0)                           (condition_1 of CW-QMIX)
// =====================================================================================================
__global__ void __launch_bounds__(256) wqmix_select_fwd_kernel(
    const float *__restrict__ q_all, const float *__restrict__ q_cent, const float *__restrict__ q_cent_tgt,
    const float *__restrict__ q_tgt, const float *__restrict__ actions, const float *__restrict__ agent_mask,
    const float *__restrict__ filled, const uint8_t *__restrict__ avail, int avail_ld, int B, int n, int T, int A,
    int double_q, float *__restrict__ q_eval_taken, float *__restrict__ q_cent_taken, float *__restrict__ q_next_cent,
    int32_t *__restrict__ greedy, uint8_t *__restrict__ agree, float *__restrict__ filled_sum,
    double *__restrict__ scratch) {
    __shared__ double red[32];
    double acc[1] = {0.0};
    const int64_t R = (int64_t)B * T;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < R; row += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(row / T), t = (int)(row % T);
        const float f = filled[row];
        bool all_agree = true;
        for (int i = 0; i < n; ++i) {
            const int64_t e = ((int64_t)b * n + i) * T + t;       // [B, n, T] element
            const int64_t s0 = ((int64_t)b * n + i) * (T + 1) + t; // [B, n, T+1] step t
            const float m = agent_mask[e] * f;
            const uint8_t *av0 = avail ? avail + s0 * avail_ld : nullptr;
            const uint8_t *av1 = avail ? av0 + avail_ld : nullptr;
            const float *qe = q_all + s0 * A;
            const int a = (int)actions[e];
            const int g = wq_argmax(qe, av0, A);
            const int an = double_q ? wq_argmax(qe + A, av1, A) : wq_argmax(q_tgt + (s0 + 1) * A, nullptr, A);
            q_eval_taken[row * n + i] = qe[a] * m;
            q_cent_taken[row * n + i] = q_cent[s0 * A + g] * m;
            q_next_cent[row * n + i] = q_cent_tgt[(s0 + 1) * A + an] * m;
            greedy[e] = g;
            all_agree = all_agree && (g == a) && (m != 0.f);
        }
        agree[row] = all_agree ? 1 : 0;
        acc[0] += (double)f;
    }
    grid_sum_finalize<1>(acc, scratch, red, [&](double(&tot)[1]) { filled_sum[0] = (float)tot[0]; });
}

// (b) backward: dq_all[b,i,t,a_t] = d_eval[row,i] * m ; dq_cent[b,i,t,g_t] = d_cent[row,i] * m (outputs pre-zeroed)
__global__ void __launch_bounds__(256) wqmix_select_bwd_kernel(const float *__restrict__ d_eval,
                                                               const float *__restrict__ d_cent,
                                                               const float *__restrict__ actions,
                                                               const int32_t *__restrict__ greedy,
                                                               const float *__restrict__ agent_mask,
                                                               const float *__restrict__ filled, int B, int n, int T,
                                                               int A, float *__restrict__ dq_all,
                                                               float *__restrict__ dq_cent) {
    const int64_t total = (int64_t)B * n * T;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int t = (int)(e % T);
        const int i = (int)((e / T) % n);
        const int b = (int)(e / ((int64_t)T * n));
        const int64_t row = (int64_t)b * T + t;
        const float m = agent_mask[e] * filled[row];
        const int64_t s0 = ((int64_t)b * n + i) * (T + 1) + t;
        if (d_eval) dq_all[s0 * A + (int)actions[e]] = d_eval[row * n + i] * m;
        if (d_cent) dq_cent[s0 * A + greedy[e]] = d_cent[row * n + i] * m;
    }
}

extern "C" int xb_wqmix_select_fwd(const float *q_all, const float *q_cent, const float *q_cent_tgt, const float *q_tgt,
                                   const float *actions, const float *agent_mask, const float *filled,
                                   const uint8_t *avail, int avail_ld, int B, int n, int T, int A, int double_q,
                                   float *q_eval_taken, float *q_cent_taken, float *q_next_cent, int32_t *greedy,
                                   uint8_t *agree, float *filled_sum, double *scratch, void *stream) {
    if (!q_all || !q_cent || !q_cent_tgt || !actions || !agent_mask || !filled || !q_eval_taken || !q_cent_taken ||
        !q_next_cent || !greedy || !agree || !filled_sum || !scratch)
        return XB_EINVAL;
    if (!double_q && !q_tgt) return XB_EINVAL;
    if (B <= 0 || n <= 0 || T <= 0 || A <= 0 || (avail && avail_ld < A)) return XB_EINVAL;
    if (n > 16) return XB_ERANGE;  // the K9 mixer's limit: these outputs feed it
    int64_t R = (int64_t)B * T, want = (R + 255) / 256;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    wqmix_select_fwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
        q_all, q_cent, q_cent_tgt, double_q ? nullptr : q_tgt, actions, agent_mask, filled, avail, avail_ld, B, n, T, A,
        double_q, q_eval_taken, q_cent_taken, q_next_cent, greedy, agree, filled_sum, scratch);
    return xb_launch_status();
}

extern "C" int xb_wqmix_select_bwd(const float *d_eval, const float *d_cent, const float *actions,
                                   const int32_t *greedy, const float *agent_mask, const float *filled, int B, int n,
                                   int T, int A, float *dq_all, float *dq_cent, void *stream) {
    if (!actions || !greedy || !agent_mask || !filled) return XB_EINVAL;
    if (!d_eval != !dq_all || !d_cent != !dq_cent || (!d_eval && !d_cent)) return XB_EINVAL;
    if (B <= 0 || n <= 0 || T <= 0 || A <= 0) return XB_EINVAL;
    if (n > 16) return XB_ERANGE;
    int64_t total = (int64_t)B * n * T, want = (total + 255) / 256;
    int64_t cap = (int64_t)xb_sm_count() * 8;
    wqmix_select_bwd_kernel<<<(int)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(
        d_eval, d_cent, actions, greedy, agent_mask, filled, B, n, T, A, dq_all, dq_cent);
    return xb_launch_status();
}

// =====================================================================================================
// (c) loss (wqmix_learner.py:141-199, use_rnn): r = mean_i rewards, d = all_i terminals,
//     y = r + (1-d)*gamma*q_ff_next ; td = q_tot - y ; w = alpha, set to 1 where (OW) td < 0 / (CW) agree | y > q_ff
//     loss_Qmix = sum(w*td^2*filled)/filled_sum ; loss_central = sum((q_ff-y)^2*filled)/filled_sum
//     dq_tot = 2*w*td*filled/filled_sum ; dq_ff = 2*(q_ff-y)*filled/filled_sum   (y and w carry no gradient)
// filled_sum and rows_total are GLOBAL, so the shards' outputs SUM to the global result (K9's contract).
// =====================================================================================================
__global__ void __launch_bounds__(256) wqmix_loss_kernel(
    const float *__restrict__ q_tot, const float *__restrict__ q_ff, const float *__restrict__ q_ff_next,
    const float *__restrict__ rewards, const float *__restrict__ terminals, const float *__restrict__ filled,
    const uint8_t *__restrict__ agree, const float *__restrict__ filled_sum, int B, int n, int T, int mode, float alpha,
    float gamma, int64_t rows_total, float *__restrict__ dq_tot, float *__restrict__ dq_ff, float *__restrict__ stats,
    double *__restrict__ scratch) {
    __shared__ double red[3 * 32];
    double acc[3] = {0, 0, 0};
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
        const float y = r_tot + (1.f - d_tot) * gamma * q_ff_next[row];
        const float qt = q_tot[row], qf = q_ff[row], f = filled[row];
        const float td = qt - y, dc = qf - y;
        const bool one = mode == XB_WQMIX_OW ? (td < 0.f) : (agree[row] != 0 || y > qf);
        const float w = one ? 1.f : alpha;
        dq_tot[row] = 2.f * w * td * f / fs;
        dq_ff[row] = 2.f * dc * f / fs;
        acc[0] += (double)w * td * td * f;
        acc[1] += (double)dc * dc * f;
        acc[2] += (double)qt;
    }
    grid_sum_finalize<3>(acc, scratch, red, [&](double(&s)[3]) {
        stats[0] = (float)(s[0] / (double)fs);             // loss_Qmix
        stats[1] = (float)(s[1] / (double)fs);             // loss_central
        stats[2] = (float)((s[0] + s[1]) / (double)fs);    // loss
        stats[3] = (float)(s[2] / (double)rows_total);     // predictQ = mean(q_tot)
    });
}

extern "C" int xb_wqmix_loss_fwd_bwd(const float *q_tot, const float *q_ff, const float *q_ff_next,
                                     const float *rewards, const float *terminals, const float *filled,
                                     const uint8_t *agree, const float *filled_sum, int B, int n, int T, int mode,
                                     float alpha, float gamma, int64_t rows_total, float *dq_tot, float *dq_ff,
                                     float *stats, double *scratch, void *stream) {
    if (!q_tot || !q_ff || !q_ff_next || !rewards || !terminals || !filled || !filled_sum || !dq_tot || !dq_ff ||
        !stats || !scratch)
        return XB_EINVAL;
    if (mode != XB_WQMIX_OW && mode != XB_WQMIX_CW) return XB_EINVAL;
    if (mode == XB_WQMIX_CW && !agree) return XB_EINVAL;
    if (B <= 0 || n <= 0 || T <= 0) return XB_EINVAL;
    if (n > 16) return XB_ERANGE;
    int64_t R = (int64_t)B * T, want = (R + 255) / 256;
    if (rows_total < R) return XB_EINVAL;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    wqmix_loss_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(q_tot, q_ff, q_ff_next, rewards, terminals, filled, agree,
                                                              filled_sum, B, n, T, mode, alpha, gamma, rows_total, dq_tot,
                                                              dq_ff, stats, scratch);
    return xb_launch_status();
}

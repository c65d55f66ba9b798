// SAC elementwise stages fused with their reductions and backward seeds (xuance/torch/learners/policy_gradient/
// sac_learner.py:52-88): actor loss, twin-critic TD backup + loss.  alpha is read from device memory (it is
// exp(log_alpha), a learnable scalar) so no host synchronisation is needed between the three optimiser steps.
#include "xb_common.cuh"

// p_loss = mean(alpha*log_pi - min(q1,q2));  torch.min backward: ties split 1/2 - 1/2.
__global__ void __launch_bounds__(256) sac_actor_kernel(const float *__restrict__ log_pi, const float *__restrict__ q1,
                                                        const float *__restrict__ q2, const float *__restrict__ alpha,
                                                        int64_t B, float inv_bt, float *__restrict__ dlog_pi,
                                                        float *__restrict__ dq1, float *__restrict__ dq2,
                                                        float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[3 * 32];
    const float a = alpha[0];
    double acc[3] = {0, 0, 0};
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const float lp = log_pi[b], x = q1[b], y = q2[b];
        const float mq = fminf(x, y);
        dlog_pi[b] = a * inv_bt;
        dq1[b] = -inv_bt * (x < y ? 1.f : (x == y ? 0.5f : 0.f));
        dq2[b] = -inv_bt * (y < x ? 1.f : (x == y ? 0.5f : 0.f));
        acc[0] += (double)(a * lp - mq);
        acc[1] += (double)mq;
        acc[2] += (double)lp;
    }
    grid_sum_finalize<3>(acc, scratch, red, [&](double(&t)[3]) {
        stats[0] = (float)(t[0] * (double)inv_bt);  // Ploss
        stats[1] = (float)(t[1] * (double)inv_bt);  // Qvalue = mean(min(q1,q2))
        stats[2] = (float)(t[2] * (double)inv_bt);  // mean(log_pi) (alpha loss needs it)
        stats[3] = 0.f;
    });
}

extern "C" int xb_sac_actor_loss(const float *log_pi, const float *q1, const float *q2, const float *alpha, int64_t B,
                                 int64_t B_total, float *dlog_pi, float *dq1, float *dq2, float *stats, double *scratch,
                                 void *stream) {
    if (!log_pi || !q1 || !q2 || !alpha || !dlog_pi || !dq1 || !dq2 || !stats || !scratch) return XB_EINVAL;
    if (B <= 0 || B_total < B) return XB_EINVAL;
    int64_t want = (B + 255) / 256;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    sac_actor_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(log_pi, q1, q2, alpha, B, 1.0f / (float)B_total, dlog_pi,
                                                             dq1, dq2, stats, scratch);
    return xb_launch_status();
}

// backup = r + (1-d)*gamma*(target_q - alpha*log_pi_next);  q_loss = mse(q1,backup) + mse(q2,backup)
__global__ void __launch_bounds__(256) sac_critic_kernel(const float *__restrict__ q1, const float *__restrict__ q2,
                                                         const float *__restrict__ target_q,
                                                         const float *__restrict__ log_pi_next,
                                                         const float *__restrict__ rew, const float *__restrict__ term,
                                                         const float *__restrict__ alpha, float gamma, int64_t B,
                                                         float inv_bt, float *__restrict__ dq1, float *__restrict__ dq2,
                                                         float *__restrict__ backup, float *__restrict__ stats,
                                                         double *__restrict__ scratch) {
    __shared__ double red[2 * 32];
    const float a = alpha[0];
    double acc[2] = {0, 0};
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const float tv = __fsub_rn(target_q[b], __fmul_rn(a, log_pi_next[b]));
        const float y = __fadd_rn(rew[b], __fmul_rn(__fmul_rn(__fsub_rn(1.f, term[b]), gamma), tv));
        backup[b] = y;
        const float e1 = q1[b] - y, e2 = q2[b] - y;
        dq1[b] = 2.f * e1 * inv_bt;
        dq2[b] = 2.f * e2 * inv_bt;
        acc[0] += (double)e1 * e1;
        acc[1] += (double)e2 * e2;
    }
    grid_sum_finalize<2>(acc, scratch, red, [&](double(&t)[2]) {
        stats[0] = (float)(t[0] * (double)inv_bt) + (float)(t[1] * (double)inv_bt);  // Qloss
        stats[1] = 0.f;
    });
}

extern "C" int xb_sac_critic_loss(const float *q1, const float *q2, const float *target_q, const float *log_pi_next,
                                  const float *rew, const float *term, const float *alpha, float gamma, int64_t B,
                                  int64_t B_total, float *dq1, float *dq2, float *backup, float *stats, double *scratch,
                                  void *stream) {
    if (!q1 || !q2 || !target_q || !log_pi_next || !rew || !term || !alpha || !dq1 || !dq2 || !backup || !stats ||
        !scratch)
        return XB_EINVAL;
    if (B <= 0 || B_total < B) return XB_EINVAL;
    int64_t want = (B + 255) / 256;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    sac_critic_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(q1, q2, target_q, log_pi_next, rew, term, alpha, gamma, B,
                                                              1.0f / (float)B_total, dq1, dq2, backup, stats, scratch);
    return xb_launch_status();
}

// =====================================================================================================
// K8D  xb_sacdis_actor_loss / xb_sacdis_critic_loss: SAC-Discrete (sacdis_learner.py:52-75)
// =====================================================================================================
// The reference's policy probabilities are Categorical(logits).probs = softmax(z - logsumexp(z)) and its log-policy is
// log(p + 1e-8 * [p == 0]) (actor_critic.py:184-205): floored only where p underflowed to exactly 0.  Subnormal p stay
// nonzero because the library is built with flush-to-zero off, as on the CPU.  One thread per row, the row in registers.

// In: the logits of a row in p[0..A).  Out: p = softmax(z - lse(z)) in torch's order (two max-shifted passes; the second
// multiplies by the reciprocal of its sum, as the CPU softmax kernel does).
template <int A_MAX>
__device__ __forceinline__ void sacdis_probs(float (&p)[A_MAX], int A) {
    float m = -INFINITY;
#pragma unroll
    for (int i = 0; i < A_MAX; ++i)
        if (i < A) m = fmaxf(m, p[i]);
    float se = 0.f;
#pragma unroll
    for (int i = 0; i < A_MAX; ++i)
        if (i < A) se = __fadd_rn(se, expf(__fsub_rn(p[i], m)));
    const float lse = __fadd_rn(logf(se), m);
    float m2 = -INFINITY;
#pragma unroll
    for (int i = 0; i < A_MAX; ++i)
        if (i < A) {
            p[i] = __fsub_rn(p[i], lse);
            m2 = fmaxf(m2, p[i]);
        }
    float s2 = 0.f;
#pragma unroll
    for (int i = 0; i < A_MAX; ++i)
        if (i < A) {
            p[i] = expf(__fsub_rn(p[i], m2));
            s2 = __fadd_rn(s2, p[i]);
        }
    const float r = __frcp_rn(s2);
#pragma unroll
    for (int i = 0; i < A_MAX; ++i)
        if (i < A) p[i] = __fmul_rn(p[i], r);
}

__device__ __forceinline__ float sacdis_log(float p) { return logf(p == 0.f ? 1e-8f : p); }  // log(p + z)

// p_loss = mean_b sum_a p*(alpha*log_pi - min(q1,q2)); dlogits = p*(g - sum p*g)/B_total with
// g_a = alpha*log_pi_a - minq_a + alpha*p_a/(p_a + z_a).  No dq: the reference's critic.zero_grad() discards it.
template <int A_MAX>
__global__ void __launch_bounds__(256, 1) sacdis_actor_kernel(const float *__restrict__ logits,
                                                              const float *__restrict__ q1,
                                                              const float *__restrict__ q2,
                                                              const float *__restrict__ alpha, int64_t B, int A,
                                                              float inv_bt, double inv_bta,
                                                              float *__restrict__ dlogits, float *__restrict__ stats,
                                                              double *__restrict__ scratch) {
    __shared__ double red[3 * 32];
    const float al = alpha[0];
    double acc[3] = {0, 0, 0};  // sum of row p_loss terms, sum min(q1,q2), sum log_pi
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const float *zr = logits + b * A, *x = q1 + b * A, *y = q2 + b * A;
        float p[A_MAX], g[A_MAX];
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) p[i] = zr[i];
        sacdis_probs<A_MAX>(p, A);
        float row = 0.f, pg = 0.f;
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) {
                const float lp = sacdis_log(p[i]), mq = fminf(x[i], y[i]);
                const float t = __fsub_rn(__fmul_rn(al, lp), mq);
                row = __fadd_rn(row, __fmul_rn(p[i], t));
                g[i] = p[i] == 0.f ? t : __fadd_rn(t, al);
                pg = __fadd_rn(pg, __fmul_rn(p[i], g[i]));
                acc[1] += (double)mq;
                acc[2] += (double)lp;
            }
        acc[0] += (double)row;
        float *dz = dlogits + b * A;
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) dz[i] = __fmul_rn(__fmul_rn(p[i], __fsub_rn(g[i], pg)), inv_bt);
    }
    grid_sum_finalize<3>(acc, scratch, red, [&](double(&t)[3]) {
        stats[0] = (float)(t[0] * (double)inv_bt);  // Ploss
        stats[1] = (float)(t[1] * inv_bta);         // Qvalue = mean(min(q1,q2)) over B_total*A
        stats[2] = (float)(t[2] * inv_bta);         // mean(log_pi) over B_total*A (the temperature step's input)
        stats[3] = 0.f;
    });
}

static inline int sacdis_grid(int64_t B) {
    const int64_t want = (B + 255) / 256;
    return (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
}

extern "C" int xb_sacdis_actor_loss(const float *logits, const float *q1, const float *q2, const float *alpha,
                                    int64_t B, int A, int64_t B_total, float *dlogits, float *stats, double *scratch,
                                    void *stream) {
    if (!logits || !q1 || !q2 || !alpha || !dlogits || !stats || !scratch) return XB_EINVAL;
    if (B <= 0 || B_total < B) return XB_EINVAL;
    if (A < 1 || A > 64) return XB_ERANGE;
    const int grid = sacdis_grid(B);
    const float inv_bt = 1.0f / (float)B_total;
    const double inv_bta = 1.0 / ((double)B_total * (double)A);
    cudaStream_t s = (cudaStream_t)stream;
#define XB_SACDIS_A(AM)                                                                                              \
    sacdis_actor_kernel<AM><<<grid, 256, 0, s>>>(logits, q1, q2, alpha, B, A, inv_bt, inv_bta, dlogits, stats, scratch)
    if (A <= 4) XB_SACDIS_A(4);
    else if (A <= 8) XB_SACDIS_A(8);
    else if (A <= 18) XB_SACDIS_A(18);
    else if (A <= 32) XB_SACDIS_A(32);
    else XB_SACDIS_A(64);
#undef XB_SACDIS_A
    return xb_launch_status();
}

// target = sum_a p'_a*(min(tq1,tq2)_a - alpha*log_pi'_a); backup = r + (1-d)*gamma*target;
// q_loss = mse(q1[a], backup) + mse(q2[a], backup).  A row whose action is not an index in [0, A) selects no column.
template <int A_MAX>
__global__ void __launch_bounds__(256, 1) sacdis_critic_kernel(
    const float *__restrict__ q1, const float *__restrict__ q2, const float *__restrict__ actions,
    const float *__restrict__ logits_next, const float *__restrict__ tq1, const float *__restrict__ tq2,
    const float *__restrict__ rew, const float *__restrict__ term, const float *__restrict__ alpha, float gamma,
    int64_t B, int A, float inv_bt, float *__restrict__ dq1, float *__restrict__ dq2, float *__restrict__ backup,
    float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[2 * 32];
    const float al = alpha[0];
    double acc[2] = {0, 0};
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const float *zr = logits_next + b * A, *x = tq1 + b * A, *y = tq2 + b * A;
        float p[A_MAX];
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) p[i] = zr[i];
        sacdis_probs<A_MAX>(p, A);
        float tv = 0.f;
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) tv = __fadd_rn(tv, __fmul_rn(p[i], __fsub_rn(fminf(x[i], y[i]), __fmul_rn(al, sacdis_log(p[i])))));
        const float bk = __fadd_rn(rew[b], __fmul_rn(__fmul_rn(__fsub_rn(1.f, term[b]), gamma), tv));
        backup[b] = bk;
        const float at = truncf(actions[b]);  // gather(act.long()): truncation toward zero
        const bool ok = at >= 0.f && at < (float)A;
        const int a = ok ? (int)at : -1;
        float e1 = __int_as_float(0x7fc00000), e2 = e1;  // NaN: the row has no selected value
        if (ok) e1 = __fsub_rn(q1[b * A + a], bk), e2 = __fsub_rn(q2[b * A + a], bk);
        float *d1 = dq1 + b * A, *d2 = dq2 + b * A;
#pragma unroll
        for (int i = 0; i < A_MAX; ++i)
            if (i < A) {
                d1[i] = i == a ? __fmul_rn(__fmul_rn(2.f, e1), inv_bt) : 0.f;
                d2[i] = i == a ? __fmul_rn(__fmul_rn(2.f, e2), inv_bt) : 0.f;
            }
        acc[0] += (double)e1 * e1;
        acc[1] += (double)e2 * e2;
    }
    grid_sum_finalize<2>(acc, scratch, red, [&](double(&t)[2]) {
        stats[0] = (float)(t[0] * (double)inv_bt) + (float)(t[1] * (double)inv_bt);  // Qloss
        stats[1] = 0.f;
    });
}

extern "C" int xb_sacdis_critic_loss(const float *q1, const float *q2, const float *actions, const float *logits_next,
                                     const float *tq1, const float *tq2, const float *rew, const float *term,
                                     const float *alpha, float gamma, int64_t B, int A, int64_t B_total, float *dq1,
                                     float *dq2, float *backup, float *stats, double *scratch, void *stream) {
    if (!q1 || !q2 || !actions || !logits_next || !tq1 || !tq2 || !rew || !term || !alpha || !dq1 || !dq2 ||
        !backup || !stats || !scratch)
        return XB_EINVAL;
    if (B <= 0 || B_total < B) return XB_EINVAL;
    if (A < 1 || A > 64) return XB_ERANGE;
    const int grid = sacdis_grid(B);
    const float inv_bt = 1.0f / (float)B_total;
    cudaStream_t s = (cudaStream_t)stream;
#define XB_SACDIS_C(AM)                                                                                              \
    sacdis_critic_kernel<AM><<<grid, 256, 0, s>>>(q1, q2, actions, logits_next, tq1, tq2, rew, term, alpha, gamma, B, \
                                                  A, inv_bt, dq1, dq2, backup, stats, scratch)
    if (A <= 4) XB_SACDIS_C(4);
    else if (A <= 8) XB_SACDIS_C(8);
    else if (A <= 18) XB_SACDIS_C(18);
    else if (A <= 32) XB_SACDIS_C(32);
    else XB_SACDIS_C(64);
#undef XB_SACDIS_C
    return xb_launch_status();
}

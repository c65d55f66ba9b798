// =====================================================================================================
// K8T  DDPG / TD3 (xuance/torch/learners/policy_gradient/{ddpg,td3}_learner.py, actor_critic.py:217-319)
// =====================================================================================================
// xb_perturb_actions: the action noise of exploration (core/off_policy.py:142-144) and of TD3's target-policy smoothing
// (TwinDelayedActorCritic.Qtarget).  xb_ddpg_critic_loss / xb_ddpg_actor_loss: the elementwise stages of both learners and
// their backward seeds, one critic (DDPG, q2 == NULL) or twin critics (TD3).  The float32 arithmetic is written with
// explicit _rn intrinsics so that nvcc cannot contract it into FMAs: the perturbed actions, the backup and the actor
// seeds are bit-identical to torch's.  Statistics are float64 partial sums through grid_sum_finalize.
#include "xb_common.cuh"

// torch.maximum / torch.minimum: a NaN in either operand is the result (fmaxf / fminf would drop it)
__device__ __forceinline__ float xb_maxn(float a, float b) { return a != a ? a : (b != b ? b : fmaxf(a, b)); }
__device__ __forceinline__ float xb_minn(float a, float b) { return a != a ? a : (b != b ? b : fminf(a, b)); }

static inline int k8t_grid(int64_t rows) {
    const int64_t want = (rows + 255) / 256;
    return (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
}

// out = clamp(a + clip(noise*scale, -noise_clip, noise_clip), low[j], high[j]), one thread per element of [B, D]
__global__ void __launch_bounds__(256) perturb_actions_kernel(const float *a, const float *__restrict__ noise,
                                                              int64_t n, int D, float scale, float noise_clip,
                                                              const float *__restrict__ low,
                                                              const float *__restrict__ high, float *out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int j = (int)(i % D);
        float e = __fmul_rn(noise[i], scale);
        if (noise_clip >= 0.f) e = xb_minn(xb_maxn(e, -noise_clip), noise_clip);
        out[i] = xb_minn(xb_maxn(__fadd_rn(a[i], e), low[j]), high[j]);
    }
}

extern "C" int xb_perturb_actions(const float *a, const float *noise, int64_t B, int D, float scale, float noise_clip,
                                  const float *low, const float *high, float *out, void *stream) {
    if (!a || !noise || !low || !high || !out) return XB_EINVAL;
    if (B <= 0 || D <= 0) return XB_EINVAL;
    const int64_t n = B * (int64_t)D;
    perturb_actions_kernel<<<k8t_grid(n), 256, 0, (cudaStream_t)stream>>>(a, noise, n, D, scale, noise_clip, low, high,
                                                                         out);
    return xb_launch_status();
}

// y = rew + (gamma*(1 - term))*t, t = tq1 or min(tq1, tq2);  q_loss = sum_i mse(q_i, y);  dq_i = 2*(q_i - y)/B_total
template <bool TWIN>
__global__ void __launch_bounds__(256) ddpg_critic_kernel(const float *__restrict__ q1, const float *__restrict__ q2,
                                                          const float *__restrict__ tq1, const float *__restrict__ tq2,
                                                          const float *__restrict__ rew,
                                                          const float *__restrict__ term, float gamma, int64_t B,
                                                          float inv_bt, float *__restrict__ dq1,
                                                          float *__restrict__ dq2, float *__restrict__ backup,
                                                          float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[4 * 32];
    double acc[4] = {0, 0, 0, 0};  // sum e1^2, sum e2^2, sum q1, sum q2
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const float t = TWIN ? xb_minn(tq1[b], tq2[b]) : tq1[b];
        const float y = __fadd_rn(rew[b], __fmul_rn(__fmul_rn(gamma, __fsub_rn(1.f, term[b])), t));
        backup[b] = y;
        const float x1 = q1[b], e1 = __fsub_rn(x1, y);
        dq1[b] = __fmul_rn(__fmul_rn(2.f, e1), inv_bt);
        acc[0] += (double)e1 * e1;
        acc[2] += (double)x1;
        if (TWIN) {
            const float x2 = q2[b], e2 = __fsub_rn(x2, y);
            dq2[b] = __fmul_rn(__fmul_rn(2.f, e2), inv_bt);
            acc[1] += (double)e2 * e2;
            acc[3] += (double)x2;
        }
    }
    grid_sum_finalize<4>(acc, scratch, red, [&](double(&s)[4]) {
        const double r = (double)inv_bt;
        stats[0] = TWIN ? __fadd_rn((float)(s[0] * r), (float)(s[1] * r)) : (float)(s[0] * r);  // Qloss
        stats[1] = (float)(s[2] * r);                                                          // mean(q1)
        stats[2] = (float)(s[3] * r);                                                          // mean(q2), 0 for DDPG
        stats[3] = 0.f;
    });
}

extern "C" int xb_ddpg_critic_loss(const float *q1, const float *q2, const float *tq1, const float *tq2,
                                   const float *rew, const float *term, float gamma, int64_t B, int64_t B_total,
                                   float *dq1, float *dq2, float *backup, float *stats, double *scratch,
                                   void *stream) {
    if (!q1 || !tq1 || !rew || !term || !dq1 || !backup || !stats || !scratch) return XB_EINVAL;
    const bool twin = q2 != nullptr;
    if ((tq2 != nullptr) != twin || (dq2 != nullptr) != twin) return XB_EINVAL;  // all three NULL or none
    if (B <= 0 || B_total < B) return XB_EINVAL;
    const float inv_bt = 1.0f / (float)B_total;
    cudaStream_t s = (cudaStream_t)stream;
    if (twin)
        ddpg_critic_kernel<true><<<k8t_grid(B), 256, 0, s>>>(q1, q2, tq1, tq2, rew, term, gamma, B, inv_bt, dq1, dq2,
                                                             backup, stats, scratch);
    else
        ddpg_critic_kernel<false><<<k8t_grid(B), 256, 0, s>>>(q1, q2, tq1, tq2, rew, term, gamma, B, inv_bt, dq1, dq2,
                                                              backup, stats, scratch);
    return xb_launch_status();
}

// DDPG: p_loss = -mean(q1), dq1 = -1/B_total.  TD3: p_loss = -mean((q1 + q2)/2), dq1 = dq2 = (-1/B_total)*0.5
template <bool TWIN>
__global__ void __launch_bounds__(256) ddpg_actor_kernel(const float *__restrict__ q1, const float *__restrict__ q2,
                                                         int64_t B, float seed, float inv_bt,
                                                         float *__restrict__ dq1, float *__restrict__ dq2,
                                                         float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[32];
    double acc[1] = {0};
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        acc[0] += TWIN ? (double)__fmul_rn(__fadd_rn(q1[b], q2[b]), 0.5f) : (double)q1[b];
        dq1[b] = seed;
        if (TWIN) dq2[b] = seed;
    }
    grid_sum_finalize<1>(acc, scratch, red, [&](double(&s)[1]) {
        stats[0] = (float)(-(s[0] * (double)inv_bt));  // Ploss
        stats[1] = stats[2] = stats[3] = 0.f;
    });
}

extern "C" int xb_ddpg_actor_loss(const float *q1, const float *q2, int64_t B, int64_t B_total, float *dq1,
                                  float *dq2, float *stats, double *scratch, void *stream) {
    if (!q1 || !dq1 || !stats || !scratch) return XB_EINVAL;
    const bool twin = q2 != nullptr;
    if ((dq2 != nullptr) != twin) return XB_EINVAL;
    if (B <= 0 || B_total < B) return XB_EINVAL;
    const float inv_bt = 1.0f / (float)B_total;
    // autograd's seed: mean's backward is -1 / numel, then the /2.0 of Qpolicy halves it (exactly)
    const float seed = -1.0f / (float)B_total;
    cudaStream_t s = (cudaStream_t)stream;
    if (twin)
        ddpg_actor_kernel<true><<<k8t_grid(B), 256, 0, s>>>(q1, q2, B, seed * 0.5f, inv_bt, dq1, dq2, stats, scratch);
    else
        ddpg_actor_kernel<false><<<k8t_grid(B), 256, 0, s>>>(q1, q2, B, seed, inv_bt, dq1, dq2, stats, scratch);
    return xb_launch_status();
}

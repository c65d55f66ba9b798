// K4C  COMA: the counterfactual critic input, the fused actor + critic loss forward / backward, and epsilon-mixed acting
// (coma_learner.py:45-137, coma_agents.py:176-273, actor_critic.py:244-324, centralized_critics.py:202-293); see
// include/xb200.h, K4C.
//
// Rows are agent steps in the episode buffer's (b, i, t) order, r = (b*n + i)*T + t.  The policy of a row is
//   p = softmax(z), z = logits with unavailable entries at -1e10 (actor_head.py:40)
//   q = (1 - eps) p + eps / A                                          (actor_critic.py:285, the epsilon mix)
//   pi = q * av / sum(q * av)   (av = 1 without an action mask: torch's Categorical(probs=q) normalisation; with one,
//                                the learner's zeroing and renormalisation, coma_learner.py:94-96)
#include "xb_common.cuh"

// ---------------------------------------------------------------- xb_coma_critic_input
// out[r] = [state(b, t) | feat[r] | joint one-hot of every agent's action at (b, t), agent i's block zeroed].  Pure
// copies and 0 / 1 constants, so the rows are bit-exact; one thread per output element.
__global__ void __launch_bounds__(256) coma_critic_input_kernel(const float *__restrict__ state,
                                                                const float *__restrict__ feat,
                                                                const float *__restrict__ actions, int64_t N, int n,
                                                                int T, int S, int F, int A, int W,
                                                                float *__restrict__ out) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < N; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / W;
        const int c = (int)(e - r * W);
        const int64_t bi = r / T;
        const int t = (int)(r - bi * T);
        const int64_t b = bi / n;
        const int i = (int)(bi - b * n);
        float v;
        if (c < S) {
            v = state[(b * T + t) * S + c];
        } else if (c < S + F) {
            v = feat[r * F + (c - S)];
        } else {
            const int k = c - S - F, j = k / A, a = k - j * A;
            v = (j != i && (int)actions[(b * n + j) * T + t] == a) ? 1.f : 0.f;
        }
        out[e] = v;
    }
}

extern "C" int xb_coma_critic_input(const float *state, const float *feat, const float *actions, int B, int n, int T,
                                    int S, int F, int A, float *out, void *stream) {
    if (!state || !feat || !actions || !out) return XB_EINVAL;
    if (B <= 0 || n <= 0 || T <= 0 || S < 0 || F < 0 || A <= 0) return XB_EINVAL;
    if (A > 64 || n > 32) return XB_ERANGE;
    const int W = S + F + n * A;
    const int64_t N = (int64_t)B * n * T * W;
    const int64_t want = (N + 255) / 256;
    const int grid = (int)(want < 65536 ? want : 65536);
    coma_critic_input_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(state, feat, actions, N, n, T, S, F, A, W, out);
    return xb_launch_status();
}

// ---------------------------------------------------------------- xb_coma_loss_fwd_bwd
// One thread per row, grid-stride; the three sums go through grid_sum_finalize (fixed order, no float atomics).
// d loss_a / d z_c = -adv * w * (1 - eps) * p_a / q_a * ([c == a] - p_c) for an available c, where a is the taken
// action and w = mask / M: the renormalisation by sum(q * av) cancels (DESIGN.md section 4).  A taken action with
// pi_a = 0 makes log pi_a = -inf and, as autograd of log(0) does, every available gradient of its row NaN.
template <int A_MAX>
__global__ void __launch_bounds__(256, 1) coma_loss_kernel(
    const float *__restrict__ logits, const uint8_t *__restrict__ avail, int avail_ld, const float *__restrict__ qv,
    const float *__restrict__ actions, const float *__restrict__ ret, const float *__restrict__ mask,
    const float *__restrict__ eps, const double *__restrict__ prep, int64_t R, int A, int64_t R_total,
    float *__restrict__ dlogits, float *__restrict__ dq, float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[3 * 32];
    double acc[3] = {0, 0, 0};  // sum -adv*log pi*mask, sum td^2, sum adv
    const double msum = prep[0];
    // the reference divides by mask.sum(): a global sum of 0 makes every weight 0/0 = NaN, as there
    const float inv_ms = (float)(1.0 / msum);
    const float e = eps[0];
    const float keep = 1.f - e, flr = e / (float)A;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
        const float *zr = logits + r * A;
        const float *qr = qv + r * A;
        const uint8_t *av = avail ? avail + r * avail_ld : nullptr;
        float z[A_MAX];
        float m = -INFINITY;
#pragma unroll
        for (int a = 0; a < A_MAX; ++a)
            if (a < A) {
                z[a] = (av && !av[a]) ? -1e10f : zr[a];
                m = fmaxf(m, z[a]);
            }
        float se = 0.f;
#pragma unroll
        for (int a = 0; a < A_MAX; ++a)
            if (a < A) se += expf(z[a] - m);
        float Z = 0.f;  // sum of q over the available actions
#pragma unroll
        for (int a = 0; a < A_MAX; ++a)
            if (a < A && !(av && !av[a])) Z += __fadd_rn(__fmul_rn(keep, expf(z[a] - m) / se), flr);
        const int act = (int)actions[r];
        float base = 0.f, p_act = 0.f, q_act = 0.f, pi_act = 0.f;
#pragma unroll
        for (int a = 0; a < A_MAX; ++a)
            if (a < A) {
                const float p = expf(z[a] - m) / se;
                const float q = __fadd_rn(__fmul_rn(keep, p), flr);
                const float pi = (av && !av[a]) ? 0.f : q / Z;
                base = __fadd_rn(base, __fmul_rn(pi, qr[a]));
                if (a == act) p_act = p, q_act = q, pi_act = pi;
            }
        const float q_taken = qr[act];
        const float adv = __fsub_rn(q_taken, base);
        const float logpi = logf(pi_act);
        const float mk = mask[r], w = mk * inv_ms;
        const float coef = pi_act > 0.f ? -adv * w * keep * p_act / q_act : NAN;
        float *dz = dlogits + r * A;
        float *dqr = dq + r * A;
        const float td = __fmul_rn(__fsub_rn(q_taken, ret[r]), mk);
#pragma unroll
        for (int a = 0; a < A_MAX; ++a)
            if (a < A) {
                const float p = expf(z[a] - m) / se;
                dz[a] = (av && !av[a]) ? 0.f : coef * ((a == act ? 1.f : 0.f) - p);
                dqr[a] = a == act ? 2.f * td * w : 0.f;
            }
        acc[0] += (double)(-adv * logpi) * (double)mk;
        acc[1] += (double)td * (double)td;
        acc[2] += (double)adv;
    }
    grid_sum_finalize<3>(acc, scratch, red, [&](double(&tt)[3]) {
        const double im = 1.0 / msum;
        stats[0] = (float)(tt[0] * im);
        stats[1] = (float)(tt[1] * im);
        stats[2] = (float)(tt[2] / (double)R_total);
        for (int k = 3; k < 8; ++k) stats[k] = 0.f;
    });
}

extern "C" int xb_coma_loss_fwd_bwd(const float *logits, const uint8_t *avail, int avail_ld, const float *q,
                                    const float *actions, const float *ret, const float *mask, const float *eps,
                                    const double *prep, int64_t R, int A, int64_t R_total, float *dlogits, float *dq,
                                    float *stats, double *scratch, void *stream) {
    if (!logits || !q || !actions || !ret || !mask || !eps || !prep || !dlogits || !dq || !stats || !scratch)
        return XB_EINVAL;
    if (R <= 0 || R_total < R || A <= 0) return XB_EINVAL;
    if (avail && avail_ld < A) return XB_EINVAL;
    if (A > 64) return XB_ERANGE;
    const int64_t want = (R + 255) / 256;
    const int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    cudaStream_t s = (cudaStream_t)stream;
#define XB_COMA(AM)                                                                                                   \
    coma_loss_kernel<AM><<<grid, 256, 0, s>>>(logits, avail, avail_ld, q, actions, ret, mask, eps, prep, R, A, R_total, \
                                              dlogits, dq, stats, scratch)
    if (A <= 4) XB_COMA(4);
    else if (A <= 8) XB_COMA(8);
    else if (A <= 18) XB_COMA(18);
    else if (A <= 32) XB_COMA(32);
    else XB_COMA(64);
#undef XB_COMA
    return xb_launch_status();
}

// ---------------------------------------------------------------- xb_coma_act
// The acting distribution pi (eps = NULL: no mix, the reference's test_mode), then the inverse CDF over pi in index
// order from u, or the first arg-max of pi (torch.argmax) without u.  Unavailable actions keep probability eps / A
// after the mix, so the draw can pick them, as the reference's Categorical(probs=q).sample() does.
template <int A_MAX>
__global__ void __launch_bounds__(128) coma_act_kernel(const float *__restrict__ logits,
                                                       const uint8_t *__restrict__ avail, int avail_ld,
                                                       const float *__restrict__ eps, const float *__restrict__ u,
                                                       int N, int A, float *__restrict__ act_f,
                                                       int32_t *__restrict__ act_i, float *__restrict__ logp) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    const float *zr = logits + (int64_t)r * A;
    const uint8_t *av = avail ? avail + (int64_t)r * avail_ld : nullptr;
    const float e = eps ? eps[0] : 0.f;
    const float keep = 1.f - e, flr = e / (float)A;
    float z[A_MAX];
    float m = -INFINITY;
#pragma unroll
    for (int a = 0; a < A_MAX; ++a)
        if (a < A) {
            z[a] = (av && !av[a]) ? -1e10f : zr[a];
            m = fmaxf(m, z[a]);
        }
    float se = 0.f;
#pragma unroll
    for (int a = 0; a < A_MAX; ++a)
        if (a < A) se += expf(z[a] - m);
    float S = 0.f;
#pragma unroll
    for (int a = 0; a < A_MAX; ++a)
        if (a < A) {
            z[a] = __fadd_rn(__fmul_rn(keep, expf(z[a] - m) / se), flr);  // z now holds q
            S += z[a];
        }
    const float uu = u ? u[r] : 0.f;
    float cdf = 0.f, best_p = -1.f, pa = 0.f, p_best = 0.f, p_last = 0.f;
    int a_s = -1, best = 0, last = A - 1;
#pragma unroll
    for (int a = 0; a < A_MAX; ++a)
        if (a < A) {
            const float pi = z[a] / S;
            if (pi > 0.f) last = a, p_last = pi;
            cdf += pi;
            if (u && a_s < 0 && uu < cdf) a_s = a, pa = pi;
            if (pi > best_p) best_p = pi, best = a, p_best = pi;
        }
    int a;
    if (!u) a = best, pa = p_best;
    else if (a_s < 0) a = last, pa = p_last;  // u >= the rounded total mass
    else a = a_s;
    if (act_f) act_f[r] = (float)a;
    if (act_i) act_i[r] = a;
    if (logp) logp[r] = logf(pa);
}

extern "C" int xb_coma_act(const float *logits, const uint8_t *avail, int avail_ld, const float *eps,
                           const float *uniforms, int N, int A, float *actions_f32, int32_t *actions_i32, float *logp,
                           void *stream) {
    if (!logits || N <= 0 || A <= 0) return XB_EINVAL;
    if (!actions_f32 && !actions_i32 && !logp) return XB_EINVAL;
    if (avail && avail_ld < A) return XB_EINVAL;
    if (A > 64) return XB_ERANGE;
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = (N + 127) / 128;
#define XB_CACT(AM)                                                                                                    \
    coma_act_kernel<AM><<<grid, 128, 0, s>>>(logits, avail, avail_ld, eps, uniforms, N, A, actions_f32, actions_i32, \
                                             logp)
    if (A <= 4) XB_CACT(4);
    else if (A <= 8) XB_CACT(8);
    else if (A <= 18) XB_CACT(18);
    else if (A <= 32) XB_CACT(32);
    else XB_CACT(64);
#undef XB_CACT
    return xb_launch_status();
}

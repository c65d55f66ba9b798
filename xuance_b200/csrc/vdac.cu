// K4V  xb_vdac_loss_fwd_bwd: the masked advantage actor-critic loss of VDAC (vdac_learner.py:24-147) and IAC
// (iac_learner.py:179-289) with the value mixing and its agent reduction fused in; see include/xb200.h, K4V.
//
// Rows are agent steps in the episode buffer's (b, i, t) order, r = (b*n + i)*T + t.  The kernel walks "units": one row
// for mode 0 (independent values), one V_tot for modes 1 and 2.  A unit u = b*T + t of the mixing modes owns the n
// loss rows paired with V_tot(u) - (b, i, t) for i < n in the aligned order, u*n + i in the reference's - so a single
// thread forms V_tot, every loss term that reads it and the sum of their gradients, in a fixed order and with no
// atomics.  Each row belongs to exactly one unit in either order, so the actor terms ride along with the critic terms.
#include "xb_common.cuh"

template <int A_MAX>
__global__ void __launch_bounds__(256, 1) vdac_loss_kernel(
    const float *__restrict__ logits, const uint8_t *__restrict__ avail, int avail_ld,
    const float *__restrict__ actions, const float *__restrict__ adv, const float *__restrict__ value,
    const float *__restrict__ old_value, const float *__restrict__ ret, const float *__restrict__ mask,
    const float *__restrict__ vn, const double *__restrict__ prep, int64_t U, int A, int n, int T, int mode,
    int row_order, int64_t R_total, float vclip, float hdelta, float vf_coef, float ent_coef,
    float *__restrict__ dlogits, float *__restrict__ dvalue, float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[4 * 32];
    double acc[4] = {0, 0, 0, 0};  // sum mask*(-adv*logp), mask*critic loss, mask*entropy, value
    const double msum = prep[0];
    // the reference divides by mask.sum(): with a global sum of 0 every weight is 0/0 = NaN, as there
    const float inv_ms = (float)(1.0 / msum);
    float vmean = 0.f, vstd = 1.f;
    if (vn) vmean = vn[0], vstd = vn[1];
    const int k = mode == 0 ? 1 : n;
    for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < U; u += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = u / T, t = u - b * T;
        float vtot = 0.f;
        if (mode == 1) {  // VDN: V_tot(b, t) = sum_i V_i, agents in index order
            for (int i = 0; i < n; ++i) vtot = __fadd_rn(vtot, value[(b * n + i) * T + t]);
        } else if (mode == 2) {
            vtot = value[u];
        }
        float dtot = 0.f;
        for (int j = 0; j < k; ++j) {
            const int64_t r = mode == 0 ? u : (row_order ? u * n + j : (b * n + j) * T + t);
            const float *zr = logits + r * A;
            const uint8_t *av = avail ? avail + r * avail_ld : nullptr;
            float z[A_MAX];
#pragma unroll
            for (int a = 0; a < A_MAX; ++a)
                if (a < A) z[a] = (av && !av[a]) ? -1e10f : zr[a];  // actor_head.py:40 (in place: no gradient there)
            float m = -INFINITY;
#pragma unroll
            for (int a = 0; a < A_MAX; ++a)
                if (a < A) m = fmaxf(m, z[a]);
            float se = 0.f;
#pragma unroll
            for (int a = 0; a < A_MAX; ++a)
                if (a < A) se += expf(z[a] - m);
            const float lse = m + logf(se);
            const int act = (int)actions[r];
            float ent = 0.f, logp_a = 0.f;
#pragma unroll
            for (int a = 0; a < A_MAX; ++a) {
                if (a < A) {
                    const float lp = z[a] - lse;
                    ent -= expf(lp) * lp;
                    if (a == act) logp_a = lp;
                }
            }
            const float mk = mask[r], w = mk * inv_ms;
            const float ad = adv[r];
            // policy: -(adv.detach() * log_pi * mask).sum() / mask.sum()
            const float d_logp = -w * ad;
            const float dent = -ent_coef * w;
            float *dz = dlogits + r * A;
#pragma unroll
            for (int a = 0; a < A_MAX; ++a) {
                if (a < A) {
                    const float lp = z[a] - lse, p = expf(lp);
                    const float g = d_logp * ((a == act ? 1.f : 0.f) - p) + dent * (-p * (lp + ent));
                    dz[a] = (av && !av[a]) ? 0.f : g;
                }
            }
            // critic: K4M's value clipping, value normalisation of the target, Huber or squared error, max of the two
            const float vp = mode == 0 ? value[r] : vtot;
            const float tgt = vn ? __fdiv_rn(__fsub_rn(ret[r], vmean), vstd) : ret[r];
            float l1, gv1, lc, dlc;
            value_loss(__fsub_rn(vp, tgt), hdelta, l1, gv1);
            if (vclip > 0.f) {
                const float vo = old_value[r];
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
            const float g = vf_coef * w * dlc;
            if (mode == 0) dvalue[r] = g;
            else dtot = __fadd_rn(dtot, g);  // the n copies of V_tot, in unit order
            acc[0] += (double)(-ad * logp_a) * (double)mk;
            acc[1] += (double)lc * (double)mk;
            acc[2] += (double)ent * (double)mk;
            acc[3] += (double)vp;
        }
        if (mode == 1) {  // dV_i = dV_tot(b, t) for every agent of the step
            for (int i = 0; i < n; ++i) dvalue[(b * n + i) * T + t] = dtot;
        } else if (mode == 2) {
            dvalue[u] = dtot;
        }
    }
    grid_sum_finalize<4>(acc, scratch, red, [&](double(&tt)[4]) {
        const double im = 1.0 / msum;
        const float a_loss = (float)(tt[0] * im), c_loss = (float)(tt[1] * im), e = (float)(tt[2] * im);
        stats[0] = a_loss;
        stats[1] = c_loss;
        stats[2] = e;
        stats[3] = (float)(tt[3] / (double)R_total);
        stats[4] = a_loss + vf_coef * c_loss - ent_coef * e;
        stats[5] = 0.f;
        stats[6] = 0.f;
        stats[7] = 0.f;
    });
}

extern "C" int xb_vdac_loss_fwd_bwd(const float *logits, const uint8_t *avail, int avail_ld, const float *actions,
                                    const float *adv, const float *value, const float *old_value, const float *ret,
                                    const float *mask, const float *vn, const double *prep, int64_t R, int A, int n,
                                    int T, int mix_mode, int row_order, int64_t R_total, float value_clip_range,
                                    float huber_delta, float vf_coef, float ent_coef, float *dlogits, float *dvalue,
                                    float *stats, double *scratch, void *stream) {
    if (!logits || !actions || !adv || !value || !ret || !mask || !prep || !dlogits || !dvalue || !stats || !scratch)
        return XB_EINVAL;
    if (value_clip_range > 0.f && !old_value) return XB_EINVAL;
    if (R <= 0 || R_total < R || A <= 0 || n <= 0 || T <= 0) return XB_EINVAL;
    if (mix_mode < 0 || mix_mode > 2 || row_order < 0 || row_order > 1) return XB_EINVAL;
    if (R % ((int64_t)n * T) != 0) return XB_EINVAL;
    if (avail && avail_ld < A) return XB_EINVAL;
    if (A > 64 || n > 32) return XB_ERANGE;
    const int64_t U = mix_mode == 0 ? R : R / n;
    const int64_t want = (U + 255) / 256;
    const int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    cudaStream_t s = (cudaStream_t)stream;
#define XB_VDAC(AM)                                                                                                  \
    vdac_loss_kernel<AM><<<grid, 256, 0, s>>>(logits, avail, avail_ld, actions, adv, value, old_value, ret, mask,   \
                                              vn, prep, U, A, n, T, mix_mode, row_order, R_total, value_clip_range,  \
                                              huber_delta, vf_coef, ent_coef, dlogits, dvalue, stats, scratch)
    if (A <= 4) XB_VDAC(4);
    else if (A <= 8) XB_VDAC(8);
    else if (A <= 18) XB_VDAC(18);
    else if (A <= 32) XB_VDAC(32);
    else XB_VDAC(64);
#undef XB_VDAC
    return xb_launch_status();
}

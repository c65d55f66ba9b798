// K9I  IQL (iql_learner.py:37-142 for use_rnn=True): (a) the global mask sum M = sum(agent_mask * filled) and (b) the
// per-agent masked double-Q TD loss with its gradient to the agent-network outputs, in one launch; see include/xb200.h,
// K9I, for the contract.
//
// (b) walks tiles of IQL_ROWS consecutive rows e = (b*n + i)*(T+1) + t1 of q_all / q_tgt [B*n*(T+1), A].  A tile stages
// its rows and the one after it through shared memory (row t+1 of one step is row t of the next, so each row is read
// once), one thread per row forms the row's loss term from shared memory, and the tile's dq rows are written back
// coalesced (every element: the gradient at the taken action, zero elsewhere and on step T).
#include "xb_common.cuh"

namespace {

constexpr int IQL_ROWS = 128;  // rows per tile = threads per CTA

__global__ void __launch_bounds__(256) iql_prepare_kernel(const float *__restrict__ agent_mask,
                                                          const float *__restrict__ filled, int n, int T, int64_t R,
                                                          double *__restrict__ msum, double *__restrict__ scratch) {
    __shared__ double red[32];
    double acc[1] = {0.0};
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < R; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t bi = e / T, t = e - bi * T, b = bi / n;
        acc[0] += (double)__fmul_rn(agent_mask[e], filled[b * T + t]);
    }
    grid_sum_finalize<1>(acc, scratch, red, [&](double(&tot)[1]) { msum[0] = tot[0]; });
}

__global__ void __launch_bounds__(IQL_ROWS) iql_td_kernel(
    const float *__restrict__ q_all, const float *__restrict__ q_tgt, const float *__restrict__ actions,
    const float *__restrict__ rewards, const float *__restrict__ terminals, const float *__restrict__ agent_mask,
    const float *__restrict__ filled, const uint8_t *__restrict__ avail, int avail_ld, const double *__restrict__ msum,
    int n, int T, int A, int double_q, float gamma, int64_t E, int64_t rows_total, float *__restrict__ dq_all,
    float *__restrict__ stats, double *__restrict__ scratch, int32_t *__restrict__ next_out,
    float *__restrict__ q_next_out, float *__restrict__ y_out) {
    extern __shared__ float sm[];
    __shared__ float s_grad[IQL_ROWS];
    __shared__ int s_act[IQL_ROWS];
    __shared__ double red[2 * 32];
    const int ld = A | 1;  // odd row stride: the thread-per-row reads below are bank-conflict free
    float *se = sm, *st = sm + (IQL_ROWS + 1) * ld;
    const int tid = threadIdx.x, T1 = T + 1;
    const float NEG = -1e10f;
    const double M = msum[0];
    // autograd of sum(td^2) / M: d/d td = (1 / M) * (2 * td), then * m through td = (q - y) * m
    const float inv = __fdiv_rn(1.f, (float)M);
    double acc[2] = {0.0, 0.0};  // sum td^2, sum q_eval_taken
    const int64_t tiles = (E + IQL_ROWS - 1) / IQL_ROWS;
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int64_t e0 = tile * IQL_ROWS;
        const int staged = (int)min((int64_t)IQL_ROWS + 1, E - e0);
        const float *ge = q_all + e0 * A, *gt = q_tgt + e0 * A;
        for (int k = tid; k < staged * A; k += IQL_ROWS) {
            const int r = k / A, c = k - r * A;
            se[r * ld + c] = ge[k];
            st[r * ld + c] = gt[k];
        }
        __syncthreads();
        const int64_t e = e0 + tid;
        float g = 0.f;
        int act = -1;
        if (e < E) {
            const int64_t s = e / T1;
            const int t = (int)(e - s * T1);
            if (t < T) {  // step T has no loss term (the reference slices it off q_eval)
                const int64_t row = s * T + t, b = s / n;
                const float *qe1 = se + (tid + 1) * ld, *qt1 = st + (tid + 1) * ld;
                const uint8_t *av = avail ? avail + (e + 1) * avail_ld : nullptr;
                // greedy next action: first maximal index of the eval values at t+1, unavailable ones at -1e10
                int best = 0;
                float bv = (av && !av[0]) ? NEG : qe1[0];
                for (int k = 1; k < A; ++k) {
                    const float v = (av && !av[k]) ? NEG : qe1[k];
                    if (v > bv) bv = v, best = k;
                }
                float qn;
                if (double_q) {
                    qn = (av && !av[best]) ? NEG : qt1[best];
                } else {
                    qn = (av && !av[0]) ? NEG : qt1[0];
                    for (int k = 1; k < A; ++k) qn = fmaxf(qn, (av && !av[k]) ? NEG : qt1[k]);
                }
                // y = r + (1 - d) * gamma * q_next, one float32 operation at a time in the reference's order
                const float y =
                    __fadd_rn(rewards[row], __fmul_rn(__fmul_rn(__fsub_rn(1.f, terminals[row]), gamma), qn));
                const float m = __fmul_rn(agent_mask[row], filled[b * T + t]);
                const int a = (int)actions[row];
                const bool ok = a >= 0 && a < A;
                const float qe = ok ? se[tid * ld + a] : __int_as_float(0x7fc00000);
                const float td = __fmul_rn(__fsub_rn(qe, y), m);
                g = __fmul_rn(__fmul_rn(inv, __fmul_rn(2.f, td)), m);
                act = ok ? a : -1;
                acc[0] += (double)__fmul_rn(td, td);
                acc[1] += (double)qe;
                if (next_out) next_out[row] = best;
                if (q_next_out) q_next_out[row] = qn;
                if (y_out) y_out[row] = y;
            }
        }
        s_grad[tid] = g;
        s_act[tid] = act;
        __syncthreads();
        const int rows = (int)min((int64_t)IQL_ROWS, E - e0);
        float *gd = dq_all + e0 * A;
        for (int k = tid; k < rows * A; k += IQL_ROWS) {
            const int r = k / A, c = k - r * A;
            gd[k] = c == s_act[r] ? s_grad[r] : 0.f;
        }
        __syncthreads();  // the next tile overwrites the staged rows
    }
    grid_sum_finalize<2>(acc, scratch, red, [&](double(&tot)[2]) {
        stats[0] = (float)(tot[0] / M);                   // loss_Q: M = 0 gives 0/0 = NaN, as the reference
        stats[1] = (float)(tot[1] / (double)rows_total);  // predictQ: the unmasked mean
    });
}

}  // namespace

extern "C" int xb_iql_prepare(const float *agent_mask, const float *filled, int B, int n, int T, double *msum,
                              double *scratch, void *stream) {
    if (!agent_mask || !filled || !msum || !scratch) return XB_EINVAL;
    if (B <= 0 || n <= 0 || T <= 0) return XB_EINVAL;
    const int64_t R = (int64_t)B * n * T, want = (R + 255) / 256;
    const int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    iql_prepare_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(agent_mask, filled, n, T, R, msum, scratch);
    return xb_launch_status();
}

extern "C" int xb_iql_td_fwd_bwd(const float *q_all, const float *q_tgt, const float *actions, const float *rewards,
                                 const float *terminals, const float *agent_mask, const float *filled,
                                 const uint8_t *avail, int avail_ld, const double *msum, int B, int n, int T, int A,
                                 int double_q, float gamma, int64_t rows_total, float *dq_all, float *stats,
                                 double *scratch, int32_t *next_actions, float *q_next, float *target, void *stream) {
    if (!q_all || !q_tgt || !actions || !rewards || !terminals || !agent_mask || !filled || !msum || !dq_all ||
        !stats || !scratch)
        return XB_EINVAL;
    if (B <= 0 || n <= 0 || T <= 0 || A <= 0 || (avail && avail_ld < A)) return XB_EINVAL;
    if (rows_total < (int64_t)B * n * T) return XB_EINVAL;
    if (A > XB_IQL_MAX_ACTIONS || n > XB_IQL_MAX_AGENTS) return XB_ERANGE;
    const int64_t E = (int64_t)B * n * (T + 1), tiles = (E + IQL_ROWS - 1) / IQL_ROWS;
    const int grid = (int)(tiles < XB_MAX_PARTIALS ? tiles : XB_MAX_PARTIALS);
    const int smem = 2 * (IQL_ROWS + 1) * (A | 1) * (int)sizeof(float);
    if (smem > 48 * 1024) {
        cudaError_t err = cudaFuncSetAttribute(iql_td_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (err != cudaSuccess) return (int)err;
    }
    iql_td_kernel<<<grid, IQL_ROWS, smem, (cudaStream_t)stream>>>(
        q_all, q_tgt, actions, rewards, terminals, agent_mask, filled, avail, avail_ld, msum, n, T, A, double_q, gamma,
        E, rows_total, dq_all, stats, scratch, next_actions, q_next, target);
    return xb_launch_status();
}

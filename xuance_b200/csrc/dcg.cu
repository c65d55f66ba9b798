// K9C Deep Coordination Graphs (DCG / DCG_S, dcg_learner.py:39-215): (a) the whole max-plus belief propagation of
// DCG_Learner.act plus its masked arg-max in ONE launch, one CTA per graph instance, (b) the coordination-graph values
// Q = sum_v u_v[a_v] + sum_e F_e[a_from, a_to] of q_dcg for the taken (eval heads) and the greedy next (target heads)
// actions, (c) the masked TD loss with dq and dV, (d) the scatter of dq into the utility and both payoff orientations.
// The utility / payoff MLPs themselves are cuBLAS GEMMs through torch; see include/xb200.h, K9C, for the contract.
//
// Arithmetic order is part of the contract (the float64 restatement in tests/dcg_refs.py is bit-exact): every add,
// subtract, multiply and divide is an explicit _rn intrinsic, so no FMA contraction can change a result.
#include "xb_common.cuh"

namespace {

constexpr int DCG_THREADS = 128;   // four warps: warps over edges in the message phase, threads over (v, a) after it

// a / b correctly rounded, from y = RN(1/b) computed on the host: q0 = RN(a*y) is faithful, the residual
// r = a - q0*b is exact in one fma, and RN(q0 + r*y) is the correctly rounded quotient (Markstein's theorem; no overflow
// or underflow for the operands here).  Bit-identical to a / b, without the call of the double-division slow path.
__device__ __forceinline__ double dcg_div(double a, double b, double y) {
    const double q0 = __dmul_rn(a, y);
    const double r = __fma_rn(-q0, b, a);
    return __fma_rn(r, y, q0);
}

// F_e[i][j] = ((P0[i*A + j] + P1[j*A + i]) / 2 in float32) / E in float64 (coordination_graph.py:87-103 then
// dcg_learner.py:54).  p0 / p1 point at the instance's edge-e row of the two orientations.
__device__ __forceinline__ double dcg_payoff(const float *__restrict__ p0, const float *__restrict__ p1, int A, int i,
                                             int j, double E, double rE) {
    const float s = __fmul_rn(__fadd_rn(__ldg(p0 + i * A + j), __ldg(p1 + j * A + i)), 0.5f);
    return dcg_div((double)s, E, rE);
}

// The payoff entries F_e[i][j] of one edge: formed from the raw orientations on every read, or (CACHE) read from the
// float64 table the CTA formed once before the iterations.  Both give the same bits.
template <bool CACHE>
struct DcgPayoffRow {
    const float *p0, *p1;   // raw orientations of this edge (CACHE = false)
    const double *Fe;       // F_e [A][A] in shared memory (CACHE = true)
    int A;
    double dE, rE;
    __device__ __forceinline__ double operator()(int i, int j) const {
        if constexpr (CACHE) return Fe[i * A + j];
        else return dcg_payoff(p0, p1, A, i, j, dE, rE);
    }
};

// The two new messages of edge e at action j (old messages in Mf / Mb, U read-only during the message phase):
//   m_fwd'[j] = max_i ((U[from][i] - m_bwd[i]) + F[i][j]),  m_bwd'[j] = max_k ((U[to][k] - m_fwd[k]) + F[j][k])
template <bool CACHE>
__device__ __forceinline__ void dcg_messages(const double *U, const double *Mf, const double *Mb,
                                             const DcgPayoffRow<CACHE> &F, int vf, int vt, int e, int j, int A,
                                             double &nf, double &nb) {
    double best = -INFINITY;   // max over a finite row: the first term always replaces it
    for (int i = 0; i < A; ++i) {
        const double x = __dadd_rn(__dsub_rn(U[vf * A + i], Mb[e * A + i]), F(i, j));
        best = x > best ? x : best;
    }
    nf = best;
    best = -INFINITY;
    for (int k = 0; k < A; ++k) {
        const double x = __dadd_rn(__dsub_rn(U[vt * A + k], Mf[e * A + k]), F(j, k));
        best = x > best ? x : best;
    }
    nb = best;
}

// (a) greedy.  Instance r = b*T + t reads step t0 + t of the [B, *, T1, *] head outputs.
//   shared: U [n*A], Mf [E*A] (from -> to, indexed by a_to), Mb [E*A] (to -> from, indexed by a_from),
//   (CACHE) F [E*A*A] formed once per instance, edges [2E]
template <bool CACHE>
__global__ void __launch_bounds__(DCG_THREADS) dcg_greedy_kernel(
    const float *__restrict__ f, const float *__restrict__ pay, int64_t pay_ld, const int32_t *__restrict__ e_from,
    const int32_t *__restrict__ e_to, const uint8_t *__restrict__ avail, int avail_ld, int T, int T1, int t0, int n,
    int A, int E, int n_iter, int normalize, double rn, double rE, double rA, int32_t *__restrict__ actions,
    double *__restrict__ U_out) {
    extern __shared__ double sm[];
    double *U = sm;
    double *Mf = U + n * A;
    double *Mb = Mf + E * A;
    double *Fs = Mb + E * A;                                   // E*A*A doubles when CACHE, else none
    int *sfrom = reinterpret_cast<int *>(Fs + (CACHE ? E * A * A : 0));
    int *sto = sfrom + E;
    const int64_t r = blockIdx.x;
    const int b = (int)(r / T), t = (int)(r % T), step = t0 + t;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const double dn = (double)n, dE = (double)E;
    const int A2 = A * A;
    const float *fb = f + ((int64_t)b * n * T1 + step) * A;   // u_v[a] = fb[v*T1*A + a] / n in float64
    const int64_t fv = (int64_t)T1 * A;
    for (int k = tid; k < E; k += blockDim.x) {
        sfrom[k] = e_from[k];
        sto[k] = e_to[k];
    }
    for (int k = tid; k < 2 * E * A; k += blockDim.x) Mf[k] = 0.0;
    for (int k = tid; k < n * A; k += blockDim.x) U[k] = __dadd_rn(__dadd_rn(dcg_div((double)__ldg(fb + (k / A) * fv + k % A), dn, rn), 0.0), 0.0);
    const int iters = E > 0 ? n_iter : 0;
    if (CACHE && iters > 0) {
        for (int k = tid; k < E * A2; k += blockDim.x) {
            const int e = k / A2, ij = k % A2;
            const float *p0 = pay + (((int64_t)b * E + e) * T1 + step) * A2;
            Fs[k] = dcg_payoff(p0, p0 + pay_ld, A, ij / A, ij % A, dE, rE);
        }
    }
    __syncthreads();
    for (int it = 0; it < iters; ++it) {
        // message phase (Jacobi): one warp owns edge e and both its directions, so it rewrites them in place
        for (int e = warp; e < E; e += nwarps) {
            const int vf = sfrom[e], vt = sto[e];
            const int64_t prow = (((int64_t)b * E + e) * T1 + step) * A2;
            const DcgPayoffRow<CACHE> F{pay + prow, pay + pay_ld + prow, Fs + (CACHE ? e * A2 : 0), A, dE, rE};
            const int j0 = lane, j1 = lane + 32;
            double nf0 = 0.0, nb0 = 0.0, nf1 = 0.0, nb1 = 0.0;
            if (j0 < A) dcg_messages(U, Mf, Mb, F, vf, vt, e, j0, A, nf0, nb0);
            if (j1 < A) dcg_messages(U, Mf, Mb, F, vf, vt, e, j1, A, nf1, nb1);
            __syncwarp();
            if (j0 < A) Mf[e * A + j0] = nf0, Mb[e * A + j0] = nb0;
            if (j1 < A) Mf[e * A + j1] = nf1, Mb[e * A + j1] = nb1;
            if (normalize) {
                __syncwarp();
                double sf = 0.0, sb = 0.0;   // the means, summed in action order
                for (int k = 0; k < A; ++k) {
                    sf = __dadd_rn(sf, Mf[e * A + k]);
                    sb = __dadd_rn(sb, Mb[e * A + k]);
                }
                const double mf = dcg_div(sf, (double)A, rA), mb = dcg_div(sb, (double)A, rA);
                __syncwarp();
                if (j0 < A) Mf[e * A + j0] = __dsub_rn(nf0, mf), Mb[e * A + j0] = __dsub_rn(nb0, mb);
                if (j1 < A) Mf[e * A + j1] = __dsub_rn(nf1, mf), Mb[e * A + j1] = __dsub_rn(nb1, mb);
            }
            __syncwarp();
        }
        __syncthreads();
        // vertex phase: U[v] = (u_v + sum_{to=v} m_fwd) + sum_{from=v} m_bwd, both sums in edge-index order from 0
        for (int k = tid; k < n * A; k += blockDim.x) {
            const int v = k / A, a = k % A;
            double sf = 0.0, sb = 0.0;
            for (int e = 0; e < E; ++e) {
                if (sto[e] == v) sf = __dadd_rn(sf, Mf[e * A + a]);
                if (sfrom[e] == v) sb = __dadd_rn(sb, Mb[e * A + a]);
            }
            U[k] = __dadd_rn(__dadd_rn(dcg_div((double)__ldg(fb + v * fv + a), dn, rn), sf), sb);
        }
        __syncthreads();
    }
    if (U_out)
        for (int k = tid; k < n * A; k += blockDim.x) U_out[r * n * A + k] = U[k];
    // masked arg-max: unavailable actions count as -1e10, the first maximal index wins (torch.argmax)
    for (int v = tid; v < n; v += blockDim.x) {
        const uint8_t *av = avail ? avail + (((int64_t)b * n + v) * T1 + step) * avail_ld : nullptr;
        int best = 0;
        double bv = (av && !av[0]) ? -1e10 : U[v * A];
        for (int a = 1; a < A; ++a) {
            const double x = (av && !av[a]) ? -1e10 : U[v * A + a];
            if (x > bv) {
                bv = x;
                best = a;
            }
        }
        actions[r * n + v] = best;
    }
}

// Q of one instance from heads at `step`: (sum_v u_v[a_v]) + (sum_e F_e[a_from][a_to]), sums in order from 0.0
template <typename Act>
__device__ __forceinline__ double dcg_q(const float *__restrict__ f, const float *__restrict__ pay, int64_t pay_ld,
                                        const int32_t *__restrict__ e_from, const int32_t *__restrict__ e_to, int b,
                                        int step, int T1, int n, int A, int E, int use_payoff, Act act) {
    const double dn = (double)n, dE = (double)E;
    double su = 0.0;
    for (int v = 0; v < n; ++v)
        su = __dadd_rn(su, __ddiv_rn((double)f[(((int64_t)b * n + v) * T1 + step) * A + act(v)], dn));
    if (!use_payoff) return su;
    double sp = 0.0;
    for (int e = 0; e < E; ++e) {
        const int64_t prow = (((int64_t)b * E + e) * T1 + step) * A * A;
        const int ai = act(e_from[e]), aj = act(e_to[e]);
        const float fij = __fmul_rn(__fadd_rn(pay[prow + ai * A + aj], pay[pay_ld + prow + aj * A + ai]), 0.5f);
        sp = __dadd_rn(sp, __ddiv_rn((double)fij, dE));
    }
    return __dadd_rn(su, sp);
}

// (b) q_eval[row] from the eval heads at step t and the taken actions, q_next[row] from the target heads at t+1 and the
//     greedy actions; filled_sum[0] = sum(filled).  One thread per (b, t) row.
__global__ void __launch_bounds__(256) dcg_q_fwd_kernel(
    const float *__restrict__ f_eval, const float *__restrict__ p_eval, int64_t p_eval_ld, const float *__restrict__ f_tgt,
    const float *__restrict__ p_tgt, int64_t p_tgt_ld, const float *__restrict__ actions,
    const int32_t *__restrict__ greedy, const float *__restrict__ filled, const int32_t *__restrict__ e_from,
    const int32_t *__restrict__ e_to, int B, int n, int T, int A, int E, int use_payoff, double *__restrict__ q_eval,
    double *__restrict__ q_next, float *__restrict__ filled_sum, double *__restrict__ scratch) {
    __shared__ double red[32];
    double acc[1] = {0.0};
    const int64_t R = (int64_t)B * T;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < R; row += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(row / T), t = (int)(row % T);
        q_eval[row] = dcg_q(f_eval, p_eval, p_eval_ld, e_from, e_to, b, t, T + 1, n, A, E, use_payoff,
                            [&](int v) { return (int)actions[((int64_t)b * n + v) * T + t]; });
        q_next[row] = dcg_q(f_tgt, p_tgt, p_tgt_ld, e_from, e_to, b, t + 1, T + 1, n, A, E, use_payoff,
                            [&](int v) { return (int)greedy[row * n + v]; });
        acc[0] += (double)filled[row];
    }
    grid_sum_finalize<1>(acc, scratch, red, [&](double(&tot)[1]) { filled_sum[0] = (float)tot[0]; });
}

// (c) TD: Q = q_eval (+ V(s)), Q' = q_next (+ V(s')); r = mean_i rewards (float32), d = all_i terminals;
//     y = r + ((1-d)*gamma in float32) * Q'; td = (Q - y) * filled; dq = 2*td*filled/filled_sum (float64), dV = float(dq)
//     stats[0] += sum(td^2)/filled_sum (loss_Q), stats[1] += sum(Q)/rows_total (predictQ, padded rows included)
__global__ void __launch_bounds__(256) dcg_td_kernel(
    const double *__restrict__ q_eval, const double *__restrict__ q_next, const float *__restrict__ v,
    const float *__restrict__ v_next, const float *__restrict__ rewards, const float *__restrict__ terminals,
    const float *__restrict__ filled, const float *__restrict__ filled_sum, int B, int n, int T, float gamma,
    int64_t rows_total, double *__restrict__ dq, float *__restrict__ dv, float *__restrict__ stats,
    double *__restrict__ scratch) {
    __shared__ double red[2 * 32];
    double acc[2] = {0.0, 0.0};
    const double fs = (double)filled_sum[0];
    const int64_t R = (int64_t)B * T;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < R; row += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(row / T), t = (int)(row % T);
        float rs = 0.f;
        bool all_term = true;
        for (int i = 0; i < n; ++i) {
            const int64_t e = ((int64_t)b * n + i) * T + t;
            rs = __fadd_rn(rs, rewards[e]);
            all_term = all_term && (terminals[e] != 0.f);
        }
        const float r_tot = __fdiv_rn(rs, (float)n);
        const float disc = __fmul_rn(all_term ? 0.f : 1.f, gamma);
        const double q = v ? __dadd_rn(q_eval[row], (double)v[row]) : q_eval[row];
        const double qn = v_next ? __dadd_rn(q_next[row], (double)v_next[row]) : q_next[row];
        const double y = __dadd_rn((double)r_tot, __dmul_rn((double)disc, qn));
        const double f = (double)filled[row];
        const double td = __dmul_rn(__dsub_rn(q, y), f);
        const double g = __ddiv_rn(__dmul_rn(__dmul_rn(2.0, td), f), fs);
        dq[row] = g;
        if (dv) dv[row] = (float)g;
        acc[0] = __dadd_rn(acc[0], __dmul_rn(td, td));
        acc[1] = __dadd_rn(acc[1], q);
    }
    grid_sum_finalize<2>(acc, scratch, red, [&](double(&s)[2]) {
        stats[0] = (float)(s[0] / fs);                    // loss_Q
        stats[1] = (float)(s[1] / (double)rows_total);    // predictQ
    });
}

// (d) df[b,v,t,a_v] = float(dq/n); dp0[b,e,t,a_from*A+a_to] = dp1[b,e,t,a_to*A+a_from] = float(dq/E)/2 (pre-zeroed)
__global__ void __launch_bounds__(256) dcg_q_bwd_kernel(const double *__restrict__ dq, const float *__restrict__ actions,
                                                        const int32_t *__restrict__ e_from,
                                                        const int32_t *__restrict__ e_to, int B, int n, int T, int A,
                                                        int E, int use_payoff, float *__restrict__ df,
                                                        float *__restrict__ dp, int64_t dp_ld) {
    const int64_t R = (int64_t)B * T;
    const int T1 = T + 1;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < R; row += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(row / T), t = (int)(row % T);
        const double g = dq[row];
        const float gu = (float)__ddiv_rn(g, (double)n);
        auto act = [&](int v) { return (int)actions[((int64_t)b * n + v) * T + t]; };
        for (int v = 0; v < n; ++v) df[(((int64_t)b * n + v) * T1 + t) * A + act(v)] = gu;
        if (!use_payoff) continue;
        const float gp = __fmul_rn((float)__ddiv_rn(g, (double)E), 0.5f);
        for (int e = 0; e < E; ++e) {
            const int ai = act(e_from[e]), aj = act(e_to[e]);
            const int64_t prow = (((int64_t)b * E + e) * T1 + t) * A * A;
            dp[prow + ai * A + aj] = gp;
            dp[dp_ld + prow + aj * A + ai] = gp;
        }
    }
}

int dcg_grid(int64_t R) {
    const int64_t want = (R + 255) / 256;
    return (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
}

}  // namespace

#define XB_DCG_CACHE_SMEM (48 * 1024)   // the cached-payoff variant stays within the default dynamic limit

static int64_t xb_dcg_greedy_smem(int n, int A, int E) {
    return (int64_t)8 * ((int64_t)n * A + 2 * (int64_t)E * A) + (int64_t)8 * E;
}

static int dcg_check_graph(int n, int A, int E) {
    if (n <= 0 || A <= 0 || E < 0) return XB_EINVAL;
    if (n > XB_DCG_MAX_AGENTS || A > XB_DCG_MAX_ACTIONS || E > XB_DCG_MAX_EDGES) return XB_ERANGE;
    if (xb_dcg_greedy_smem(n, A, E) > XB_DCG_MAX_SMEM) return XB_ERANGE;
    return XB_OK;
}

extern "C" int xb_dcg_greedy(const float *f, const float *payoff, int64_t payoff_ld, const int32_t *edges_from,
                             const int32_t *edges_to, const uint8_t *avail, int avail_ld, int B, int T, int T1, int t0,
                             int n, int A, int E, int n_iter, int normalize, int32_t *actions, double *U_out,
                             void *stream) {
    if (!f || !actions) return XB_EINVAL;
    if (E > 0 && (!payoff || !edges_from || !edges_to || payoff_ld < (int64_t)B * E * T1 * A * A)) return XB_EINVAL;
    if (B <= 0 || T <= 0 || t0 < 0 || T1 < t0 + T || n_iter < 0 || (avail && avail_ld < A)) return XB_EINVAL;
    int rc = dcg_check_graph(n, A, E);
    if (rc != XB_OK) return rc;
    const int64_t R = (int64_t)B * T;
    if (R > 0x7fffffff) return XB_ERANGE;
    // F_e is the same in every iteration: form it once in shared memory when the table fits the cache budget
    const int64_t smem_f = xb_dcg_greedy_smem(n, A, E) + (int64_t)8 * E * A * A;
    const bool cache = E > 0 && n_iter > 1 && smem_f <= XB_DCG_CACHE_SMEM;
    const int smem = (int)(cache ? smem_f : xb_dcg_greedy_smem(n, A, E));
    const double rn = 1.0 / n, rE = E > 0 ? 1.0 / E : 0.0, rA = 1.0 / A;
    cudaStream_t st = (cudaStream_t)stream;
    if (cache) {
        dcg_greedy_kernel<true><<<(unsigned)R, DCG_THREADS, smem, st>>>(
            f, payoff, payoff_ld, edges_from, edges_to, avail, avail_ld, T, T1, t0, n, A, E, n_iter, normalize, rn, rE,
            rA, actions, U_out);
    } else {
        if (smem > 48 * 1024) {
            cudaError_t err = cudaFuncSetAttribute(dcg_greedy_kernel<false>,
                                                   cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
            if (err != cudaSuccess) return (int)err;
        }
        dcg_greedy_kernel<false><<<(unsigned)R, DCG_THREADS, smem, st>>>(
            f, payoff, payoff_ld, edges_from, edges_to, avail, avail_ld, T, T1, t0, n, A, E, n_iter, normalize, rn, rE,
            rA, actions, U_out);
    }
    return xb_launch_status();
}

extern "C" int xb_dcg_q_fwd(const float *f_eval, const float *p_eval, int64_t p_eval_ld, const float *f_tgt,
                            const float *p_tgt, int64_t p_tgt_ld, const float *actions, const int32_t *greedy,
                            const float *filled, const int32_t *edges_from, const int32_t *edges_to, int B, int n,
                            int T, int A, int E, int use_payoff, double *q_eval, double *q_next, float *filled_sum,
                            double *scratch, void *stream) {
    if (!f_eval || !f_tgt || !actions || !greedy || !filled || !q_eval || !q_next || !filled_sum || !scratch)
        return XB_EINVAL;
    if (B <= 0 || T <= 0) return XB_EINVAL;
    int rc = dcg_check_graph(n, A, E);
    if (rc != XB_OK) return rc;
    use_payoff = use_payoff && E > 0;
    const int64_t need = (int64_t)B * E * (T + 1) * A * A;
    if (use_payoff && (!p_eval || !p_tgt || !edges_from || !edges_to || p_eval_ld < need || p_tgt_ld < need))
        return XB_EINVAL;
    dcg_q_fwd_kernel<<<dcg_grid((int64_t)B * T), 256, 0, (cudaStream_t)stream>>>(
        f_eval, p_eval, p_eval_ld, f_tgt, p_tgt, p_tgt_ld, actions, greedy, filled, edges_from, edges_to, B, n, T, A, E,
        use_payoff, q_eval, q_next, filled_sum, scratch);
    return xb_launch_status();
}

extern "C" int xb_dcg_td_fwd_bwd(const double *q_eval, const double *q_next, const float *v, const float *v_next,
                                 const float *rewards, const float *terminals, const float *filled,
                                 const float *filled_sum, int B, int n, int T, float gamma, int64_t rows_total,
                                 double *dq, float *dv, float *stats, double *scratch, void *stream) {
    if (!q_eval || !q_next || !rewards || !terminals || !filled || !filled_sum || !dq || !stats || !scratch)
        return XB_EINVAL;
    if (!v != !v_next || !v != !dv) return XB_EINVAL;   // DCG_S passes V(s), V(s') and dV together
    if (B <= 0 || n <= 0 || T <= 0) return XB_EINVAL;
    if (n > XB_DCG_MAX_AGENTS) return XB_ERANGE;
    const int64_t R = (int64_t)B * T;
    if (rows_total < R) return XB_EINVAL;
    dcg_td_kernel<<<dcg_grid(R), 256, 0, (cudaStream_t)stream>>>(q_eval, q_next, v, v_next, rewards, terminals, filled,
                                                                 filled_sum, B, n, T, gamma, rows_total, dq, dv, stats,
                                                                 scratch);
    return xb_launch_status();
}

extern "C" int xb_dcg_q_bwd(const double *dq, const float *actions, const int32_t *edges_from, const int32_t *edges_to,
                            int B, int n, int T, int A, int E, int use_payoff, float *df, float *dp, int64_t dp_ld,
                            void *stream) {
    if (!dq || !actions || !df) return XB_EINVAL;
    if (B <= 0 || T <= 0) return XB_EINVAL;
    int rc = dcg_check_graph(n, A, E);
    if (rc != XB_OK) return rc;
    use_payoff = use_payoff && E > 0;
    if (use_payoff && (!dp || !edges_from || !edges_to || dp_ld < (int64_t)B * E * (T + 1) * A * A)) return XB_EINVAL;
    const int64_t R = (int64_t)B * T, want = (R + 255) / 256, cap = (int64_t)xb_sm_count() * 8;
    dcg_q_bwd_kernel<<<(int)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(
        dq, actions, edges_from, edges_to, B, n, T, A, E, use_payoff, df, dp, dp_ld);
    return xb_launch_status();
}

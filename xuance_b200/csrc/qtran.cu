// K9Q QTRAN (QTRAN_base / QTRAN_alt, qtran_learner.py:199-371): (a) the masked greedy and next actions of the eval and
// target heads, (b) the whole action-encoding input assembly of Q_tran (mask, one-hot, the shared two-layer encoder,
// the sum over agents or alt's (n-1)-fold sums, the state and agent-id columns) in one launch, (c) its backward down
// to the GRU outputs and the encoder's weights with a fixed-order reduction, (d) the TD, opt and nopt losses with every
// gradient they send to Q_jt, V_jt and the agents' heads.  Q_jt and V_jt are cuBLAS GEMMs through torch; see
// include/xb200.h, K9Q, for the contract.
#include "xb_common.cuh"

namespace {

constexpr int QT_THREADS = 128;   // >= D = H + A <= 128: thread j owns encoder unit j
constexpr int QT_PTILE = 8;       // weight-gradient rows per CTA
constexpr int QT_RTILE = 16;      // agent-rows staged per weight-gradient step
constexpr int QT_CHUNK = 128;     // least agent-rows per weight-gradient partial
constexpr int QT_MAX_CHUNKS = 1024;   // most partials: the chunk grows beyond 128*1024 agent-rows
constexpr int QT_WG_THREADS = 256;
constexpr int QT_WG_ENTRIES = (2 * QT_PTILE * 128 + 2 * QT_PTILE + QT_WG_THREADS - 1) / QT_WG_THREADS;

// The action of agent i at step t: float32 taken actions or int32 greedy / next actions, [B, n, act_T].
struct QtAct {
    const float *f;
    const int32_t *i;
    int ld;
    __device__ __forceinline__ int operator()(int b, int n, int agent, int t) const {
        const int64_t e = ((int64_t)b * n + agent) * ld + t;
        return f ? (int)f[e] : i[e];
    }
};

// first maximal index of q[0..A) with unavailable actions (av[a] == 0) at -1e10
__device__ __forceinline__ int qt_argmax(const float *__restrict__ q, const uint8_t *__restrict__ av, int A) {
    int best = 0;
    float bv = (av && !av[0]) ? -1e10f : q[0];
    for (int a = 1; a < A; ++a) {
        const float x = (av && !av[a]) ? -1e10f : q[a];
        if (x > bv) {
            bv = x;
            best = a;
        }
    }
    return best;
}

// (a) one thread per (b, i, t1), t1 in 0..T: greedy[b,i,t1] from q_all; next[b,i,t1-1] = greedy (double_q) or the masked
//     arg-max of q_tgt at t1; filled_sum[0] = sum(filled)
__global__ void __launch_bounds__(256) qtran_select_kernel(
    const float *__restrict__ q_all, const float *__restrict__ q_tgt, const uint8_t *__restrict__ avail, int avail_ld,
    const float *__restrict__ filled, int B, int n, int T, int A, int double_q, int32_t *__restrict__ greedy,
    int32_t *__restrict__ next, float *__restrict__ filled_sum, double *__restrict__ scratch) {
    __shared__ double red[32];
    double acc[1] = {0.0};
    const int T1 = T + 1;
    const int64_t N = (int64_t)B * n * T1;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < N; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t bi = e / T1;
        const int t1 = (int)(e % T1), i = (int)(bi % n), b = (int)(bi / n);
        const uint8_t *av = avail ? avail + e * avail_ld : nullptr;
        const int g = qt_argmax(q_all + e * A, av, A);
        greedy[e] = g;
        if (t1 >= 1) next[bi * T + t1 - 1] = double_q ? g : qt_argmax(q_tgt + e * A, av, A);
        if (i == 0 && t1 < T) acc[0] += (double)filled[(int64_t)b * T + t1];
    }
    grid_sum_finalize<1>(acc, scratch, red, [&](double(&tot)[1]) { filled_sum[0] = (float)tot[0]; });
}

// (b) persistent CTAs over rows r = b*T + t.  shared: W1^T, W2^T [D*D] (unit-minor, conflict-free), b1, b2, u (the
//     masked h), s1 (relu), E [n*D] (every agent's encoding of this row)
template <int MODE>
__global__ void __launch_bounds__(QT_THREADS) qtran_encode_fwd_kernel(
    const float *__restrict__ state, int state_t0, const float *__restrict__ h, const float *__restrict__ agent_mask,
    QtAct act, const float *__restrict__ w1, const float *__restrict__ b1, const float *__restrict__ w2,
    const float *__restrict__ b2, int B, int n, int T, int S, int H, int A, float *__restrict__ x,
    float *__restrict__ pre) {
    extern __shared__ float sm[];
    const int D = H + A, T1 = T + 1, tid = threadIdx.x;
    float *W1t = sm, *W2t = W1t + D * D, *sb1 = W2t + D * D, *sb2 = sb1 + D, *u = sb2 + D, *s1 = u + D, *E = s1 + D;
    for (int k = tid; k < D * D; k += blockDim.x) {
        const int j = k / D, c = k % D;
        W1t[c * D + j] = w1[k];
        W2t[c * D + j] = w2[k];
    }
    for (int k = tid; k < D; k += blockDim.x) sb1[k] = b1[k], sb2[k] = b2[k];
    __syncthreads();
    const int64_t R = (int64_t)B * T;
    const int W = S + D + (MODE == XB_QTRAN_ALT ? n : 0);
    for (int64_t r = blockIdx.x; r < R; r += gridDim.x) {
        const int b = (int)(r / T), t = (int)(r % T);
        for (int i = 0; i < n; ++i) {
            const float m = agent_mask[((int64_t)b * n + i) * T + t];
            const int a = act(b, n, i, t);
            for (int k = tid; k < H; k += blockDim.x) u[k] = __fmul_rn(h[(((int64_t)b * n + i) * T1 + t) * H + k], m);
            __syncthreads();
            if (tid < D) {
                float z = 0.f;
                for (int k = 0; k < H; ++k) z = __fmaf_rn(W1t[k * D + tid], u[k], z);
                const float oh = (unsigned)a < (unsigned)A ? W1t[(H + a) * D + tid] : 0.f;   // no read past W1^T
                z = __fadd_rn(__fadd_rn(z, oh), sb1[tid]);   // the one-hot column, then the bias
                if (pre) pre[(r * n + i) * D + tid] = z;
                s1[tid] = fmaxf(z, 0.f);
            }
            __syncthreads();
            if (tid < D) {
                float e = 0.f;
                for (int k = 0; k < D; ++k) e = __fmaf_rn(W2t[k * D + tid], s1[k], e);
                E[i * D + tid] = __fadd_rn(e, sb2[tid]);
            }
            __syncthreads();
        }
        const float *st = state + ((int64_t)b * T1 + state_t0 + t) * S;
        if (MODE == XB_QTRAN_BASE) {
            float *xr = x + r * W;
            for (int c = tid; c < W; c += blockDim.x) {
                float v;
                if (c < S) {
                    v = st[c];
                } else {
                    v = 0.f;
                    for (int i = 0; i < n; ++i) v = __fadd_rn(v, E[i * D + c - S]);
                }
                xr[c] = v;
            }
        } else {
            for (int k = tid; k < n * W; k += blockDim.x) {
                const int i = k / W, c = k % W;
                float v;
                if (c < S) {
                    v = st[c];
                } else if (c < S + D) {
                    v = 0.f;
                    for (int j = 0; j < n; ++j)   // q_mix_head.py:283-285 masks the repeat of e_i itself
                        if (j != i) v = __fadd_rn(v, E[i * D + c - S]);
                } else {
                    v = (c - S - D == i) ? 1.f : 0.f;
                }
                x[(r * n + i) * W + c] = v;
            }
        }
        __syncthreads();
    }
}

// (c1) per agent-row (r, j): ge = the encoding gradient that reaches agent j (alt: n-1 adds of its own row's), dz1 = (W2^T ge) * (z1 > 0),
//      dh = m * (W1[:, :H]^T dz1).  ge and dz1 go to the workspace for (c2).  shared: W1, W2 [D*D] row-major, G [n*D]
//      (the row's dx encoding columns), ge, dz [D]
template <int MODE>
__global__ void __launch_bounds__(QT_THREADS) qtran_encode_bwd_rows_kernel(
    const float *__restrict__ dx, int ldx, const float *__restrict__ agent_mask, const float *__restrict__ w1,
    const float *__restrict__ w2, const float *__restrict__ pre, int B, int n, int T, int S, int H, int A,
    float *__restrict__ dh, float *__restrict__ GE, float *__restrict__ DZ) {
    extern __shared__ float sm[];
    const int D = H + A, T1 = T + 1, tid = threadIdx.x;
    const int NG = MODE == XB_QTRAN_ALT ? n : 1;
    float *W1 = sm, *W2 = W1 + D * D, *G = W2 + D * D, *ge = G + NG * D, *dz = ge + D;
    for (int k = tid; k < D * D; k += blockDim.x) W1[k] = w1[k], W2[k] = w2[k];
    const int64_t R = (int64_t)B * T;
    for (int64_t r = blockIdx.x; r < R; r += gridDim.x) {
        const int b = (int)(r / T), t = (int)(r % T);
        for (int k = tid; k < NG * D; k += blockDim.x) G[k] = dx[(r * NG + k / D) * ldx + S + k % D];
        __syncthreads();
        for (int j = 0; j < n; ++j) {
            const int64_t rj = r * n + j;
            if (tid < D) {
                float g;
                if (MODE == XB_QTRAN_BASE) {
                    g = G[tid];
                } else {
                    g = 0.f;
                    for (int i = 0; i < n; ++i)
                        if (i != j) g = __fadd_rn(g, G[j * D + tid]);
                }
                ge[tid] = g;
                GE[rj * D + tid] = g;
            }
            __syncthreads();
            if (tid < D) {
                float s = 0.f;
                for (int p = 0; p < D; ++p) s = __fmaf_rn(W2[p * D + tid], ge[p], s);
                const float d = pre[rj * D + tid] > 0.f ? s : 0.f;
                dz[tid] = d;
                DZ[rj * D + tid] = d;
            }
            __syncthreads();
            const float m = agent_mask[((int64_t)b * n + j) * T + t];
            float *dhr = dh + (((int64_t)b * n + j) * T1 + t) * H;
            for (int k = tid; k < H; k += blockDim.x) {
                float s = 0.f;
                for (int p = 0; p < D; ++p) s = __fmaf_rn(W1[p * D + k], dz[p], s);
                dhr[k] = __fmul_rn(s, m);
                if (t == T - 1) dhr[H + k] = 0.f;   // step T feeds no encoding
            }
            __syncthreads();
        }
    }
}

// (c2) grid (chunk c, unit tile): the partial sums over agent-rows [c*chunk, (c+1)*chunk), in row order, of
//      dW1[p,:] += dz1[p] * u, dW2[p,:] += ge[p] * relu(z1), db1[p] += dz1[p], db2[p] += ge[p]; u = [h*m, onehot(a)], so
//      the one-hot columns take dz1 at the action and exact zeros elsewhere.  partial layout: dW1, db1, dW2, db2.
__global__ void __launch_bounds__(QT_WG_THREADS) qtran_encode_wgrad_kernel(
    const float *__restrict__ h, const float *__restrict__ agent_mask, QtAct act, const float *__restrict__ pre,
    const float *__restrict__ GE, const float *__restrict__ DZ, int B, int n, int T, int H, int A, int64_t chunk,
    float *__restrict__ partial) {
    __shared__ float U[QT_RTILE][128], S1[QT_RTILE][128], Z[QT_RTILE][128], G[QT_RTILE][128];
    const int D = H + A, T1 = T + 1, tid = threadIdx.x;
    const int64_t Rn = (int64_t)B * T * n;
    const int64_t lo = (int64_t)blockIdx.x * chunk, hi = lo + chunk < Rn ? lo + chunk : Rn;
    const int p0 = blockIdx.y * QT_PTILE, P = D - p0 < QT_PTILE ? D - p0 : QT_PTILE;
    const int NE = 2 * P * D + 2 * P;
    float acc[QT_WG_ENTRIES];
#pragma unroll
    for (int s = 0; s < QT_WG_ENTRIES; ++s) acc[s] = 0.f;
    for (int64_t r0 = lo; r0 < hi; r0 += QT_RTILE) {
        const int nr = hi - r0 < QT_RTILE ? (int)(hi - r0) : QT_RTILE;
        for (int k = tid; k < nr * D; k += blockDim.x) {
            const int rr = k / D, c = k % D;
            const int64_t rj = r0 + rr;
            const int j = (int)(rj % n);
            const int64_t r = rj / n;
            const int b = (int)(r / T), t = (int)(r % T);
            float uv;
            if (c < H) uv = __fmul_rn(h[(((int64_t)b * n + j) * T1 + t) * H + c], agent_mask[((int64_t)b * n + j) * T + t]);
            else uv = (c - H == act(b, n, j, t)) ? 1.f : 0.f;
            U[rr][c] = uv;
            S1[rr][c] = fmaxf(pre[rj * D + c], 0.f);
            Z[rr][c] = DZ[rj * D + c];
            G[rr][c] = GE[rj * D + c];
        }
        __syncthreads();
#pragma unroll
        for (int s = 0; s < QT_WG_ENTRIES; ++s) {
            const int e = tid + s * QT_WG_THREADS;
            if (e >= NE) continue;
            float a = acc[s];
            if (e < P * D) {
                const int p = p0 + e / D, c = e % D;
                for (int rr = 0; rr < nr; ++rr) a = __fmaf_rn(Z[rr][p], U[rr][c], a);
            } else if (e < 2 * P * D) {
                const int p = p0 + (e - P * D) / D, c = (e - P * D) % D;
                for (int rr = 0; rr < nr; ++rr) a = __fmaf_rn(G[rr][p], S1[rr][c], a);
            } else if (e < 2 * P * D + P) {
                const int p = p0 + e - 2 * P * D;
                for (int rr = 0; rr < nr; ++rr) a = __fadd_rn(a, Z[rr][p]);
            } else {
                const int p = p0 + e - 2 * P * D - P;
                for (int rr = 0; rr < nr; ++rr) a = __fadd_rn(a, G[rr][p]);
            }
            acc[s] = a;
        }
        __syncthreads();
    }
    float *out = partial + (int64_t)blockIdx.x * (2 * D * D + 2 * D);
#pragma unroll
    for (int s = 0; s < QT_WG_ENTRIES; ++s) {
        const int e = tid + s * QT_WG_THREADS;
        if (e >= NE) continue;
        int o;
        if (e < P * D) o = (p0 + e / D) * D + e % D;                                          // dW1
        else if (e < 2 * P * D) o = D * D + D + (p0 + (e - P * D) / D) * D + (e - P * D) % D;  // dW2
        else if (e < 2 * P * D + P) o = D * D + p0 + e - 2 * P * D;                            // db1
        else o = 2 * D * D + D + p0 + e - 2 * P * D - P;                                       // db2
        out[o] = acc[s];
    }
}

// (c3) every gradient entry: the sum of the chunks' partials in chunk order
__global__ void __launch_bounds__(256) qtran_encode_wsum_kernel(const float *__restrict__ partial, int nc, int D,
                                                                float *__restrict__ dw1, float *__restrict__ db1,
                                                                float *__restrict__ dw2, float *__restrict__ db2) {
    const int NP = 2 * D * D + 2 * D;
    for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < NP; o += gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int c = 0; c < nc; ++c) s = __fadd_rn(s, partial[(int64_t)c * NP + o]);
        if (o < D * D) dw1[o] = s;
        else if (o < D * D + D) db1[o - D * D] = s;
        else if (o < 2 * D * D + D) dw2[o - D * D - D] = s;
        else db2[o - 2 * D * D - D] = s;
    }
}

// (d) one thread per row r = b*T + t; float64 throughout, float32 outputs.  den = filled_sum (base) or n*filled_sum (alt)
template <int MODE>
__global__ void __launch_bounds__(256, 1) qtran_loss_kernel(
    const float *__restrict__ q_all, const float *__restrict__ actions, const int32_t *__restrict__ greedy,
    const int32_t *__restrict__ next, const float *__restrict__ agent_mask, const float *__restrict__ filled,
    const float *__restrict__ rewards, const float *__restrict__ terminals, const float *__restrict__ qjt,
    const float *__restrict__ qjt_greedy, const float *__restrict__ qjt_next, const float *__restrict__ v,
    const float *__restrict__ filled_sum, int B, int n, int T, int A, float gamma, float lambda_opt,
    float lambda_nopt, int64_t rows_total, float *__restrict__ dqjt, float *__restrict__ dv,
    float *__restrict__ dq_all, float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[4 * 32];
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    const int T1 = T + 1;
    const double den = (MODE == XB_QTRAN_ALT ? (double)n : 1.0) * (double)filled_sum[0];
    const double lo = (double)lambda_opt, ln = (double)lambda_nopt;
    const int64_t R = (int64_t)B * T;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < R; row += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(row / T), t = (int)(row % T);
        float rs = 0.f;
        bool all_term = true;
        double qtot = 0.0, qtot_g = 0.0;
        for (int i = 0; i < n; ++i) {
            const int64_t e = ((int64_t)b * n + i) * T + t;
            rs += rewards[e];
            all_term = all_term && (terminals[e] != 0.f);
            const float *qi = q_all + (((int64_t)b * n + i) * T1 + t) * A;
            const double m = (double)agent_mask[e];
            qtot += (double)qi[(int)actions[e]] * m;
            qtot_g += (double)qi[greedy[((int64_t)b * n + i) * T1 + t]] * m;
        }
        const double r_tot = (double)(rs / (float)n);
        const double disc = all_term ? 0.0 : (double)gamma;
        const double f = (double)filled[row], V = (double)v[row];
        if (MODE == XB_QTRAN_BASE) {
            const double q = (double)qjt[row];
            const double y = r_tot + disc * (double)qjt_next[row];
            const double td = (q - y) * f;
            const double eo = (qtot_g - (double)qjt_greedy[row] + V) * f;
            const double xn = qtot - q + V;
            const double en = (xn < 0.0 ? xn : 0.0) * f;
            const double c_o = lo * 2.0 * eo * f / den, c_n = ln * 2.0 * en * f / den;
            dqjt[row] = (float)(2.0 * td * f / den);
            dv[row] = (float)(c_o + c_n);
            for (int j = 0; j < n; ++j) {
                const int64_t e = ((int64_t)b * n + j) * T + t;
                const double m = (double)agent_mask[e];
                float *dqj = dq_all + (((int64_t)b * n + j) * T1 + t) * A;
                const int a = (int)actions[e], g = greedy[((int64_t)b * n + j) * T1 + t];
                if (a == g) {
                    dqj[a] = (float)((c_n + c_o) * m);
                } else {
                    dqj[a] = (float)(c_n * m);
                    dqj[g] = (float)(c_o * m);
                }
            }
            acc[0] += td * td;
            acc[1] += eo * eo;
            acc[2] += en * en;
            acc[3] += q;
        } else {
            // Q_alt rows are (row, i): qjt [R*n, A]; leave-one-out sums of the masked taken values
            double dV = 0.0, c_o_sum = 0.0;
            for (int i = 0; i < n; ++i) {
                const int64_t e = ((int64_t)b * n + i) * T + t, ri = row * n + i;
                const float *qi = q_all + (((int64_t)b * n + i) * T1 + t) * A;
                const int a = (int)actions[e], g = greedy[((int64_t)b * n + i) * T1 + t];
                const double q = (double)qjt[ri * A + a];
                const double y = r_tot + disc * (double)qjt_next[ri * A + next[e]];
                const double td = (q - y) * f;
                const double eo = (qtot_g - (double)qjt_greedy[ri * A + g] + V) * f;
                double others = 0.0;
                for (int j = 0; j < n; ++j)
                    if (j != i) {
                        const int64_t ej = ((int64_t)b * n + j) * T + t;
                        others += (double)q_all[(((int64_t)b * n + j) * T1 + t) * A + (int)actions[ej]] *
                                  (double)agent_mask[ej];
                    }
                int amin = 0;
                double xmin = (double)qi[0] + others - (double)qjt[ri * A] + V;
                for (int k = 1; k < A; ++k) {
                    const double xk = (double)qi[k] + others - (double)qjt[ri * A + k] + V;
                    if (xk < xmin) xmin = xk, amin = k;
                }
                const double en = xmin * f;
                const double c_o = lo * 2.0 * eo * f / den, c_n = ln * 2.0 * en * f / den;
                for (int k = 0; k < A; ++k) dqjt[ri * A + k] = k == a ? (float)(2.0 * td * f / den) : 0.f;
                dV += c_o + c_n;
                c_o_sum += c_o;
                // nopt reaches q[i, amin] and, through the leave-one-out sum, every other agent's masked taken value
                dq_all[(((int64_t)b * n + i) * T1 + t) * A + amin] += (float)c_n;
                for (int j = 0; j < n; ++j)
                    if (j != i) {
                        const int64_t ej = ((int64_t)b * n + j) * T + t;
                        dq_all[(((int64_t)b * n + j) * T1 + t) * A + (int)actions[ej]] += (float)(c_n * (double)agent_mask[ej]);
                    }
                acc[0] += td * td;
                acc[1] += eo * eo;
                acc[2] += en * en;
                acc[3] += q;
            }
            dv[row] = (float)dV;
            // opt: Q_tot(greedy) sends sum_i c_o(i) to every agent's masked greedy value
            for (int j = 0; j < n; ++j) {
                const int64_t e = ((int64_t)b * n + j) * T + t;
                dq_all[(((int64_t)b * n + j) * T1 + t) * A + greedy[((int64_t)b * n + j) * T1 + t]] +=
                    (float)(c_o_sum * (double)agent_mask[e]);
            }
        }
    }
    grid_sum_finalize<4>(acc, scratch, red, [&](double(&s)[4]) {
        const double l_td = s[0] / den, l_opt = s[1] / den, l_nopt = s[2] / den;
        stats[0] = (float)l_td;
        stats[1] = (float)l_opt;
        stats[2] = (float)l_nopt;
        stats[3] = (float)(l_td + lo * l_opt + ln * l_nopt);
        stats[4] = (float)(s[3] / ((double)rows_total * (MODE == XB_QTRAN_ALT ? n : 1)));   // Q_joint
    });
}

int qt_grid(int64_t R) {
    const int64_t want = (R + 255) / 256;
    return (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
}

int qt_check(int B, int n, int T, int A) {
    if (B <= 0 || n <= 0 || T <= 0 || A <= 0) return XB_EINVAL;
    if (n > XB_QTRAN_MAX_AGENTS || A > XB_QTRAN_MAX_ACTIONS) return XB_ERANGE;
    if ((int64_t)B * T * n > 0x7fffffff) return XB_ERANGE;
    return XB_OK;
}

int qt_check_enc(int mode, int B, int n, int T, int S, int H, int A) {
    if (mode != XB_QTRAN_BASE && mode != XB_QTRAN_ALT) return XB_EINVAL;
    if (S <= 0 || H <= 0) return XB_EINVAL;
    if (H > XB_QTRAN_MAX_HIDDEN) return XB_ERANGE;
    return qt_check(B, n, T, A);
}

// dynamic shared memory beyond the default 48 KB must be granted per kernel (as xb_dcg_greedy does)
template <typename K>
int qt_allow_smem(K kernel, int smem) {
    if (smem <= 48 * 1024) return XB_OK;
    cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    return err == cudaSuccess ? XB_OK : (int)err;
}

int qt_persistent_grid(int64_t R, int smem) {
    const int per_sm = smem > 0 ? (int)((200 * 1024) / smem) : 8;
    const int64_t cap = (int64_t)xb_sm_count() * (per_sm < 1 ? 1 : per_sm > 8 ? 8 : per_sm);
    return (int)(R < cap ? R : cap);
}

}  // namespace

extern "C" int xb_qtran_select(const float *q_all, const float *q_tgt, const uint8_t *avail, int avail_ld,
                               const float *filled, int B, int n, int T, int A, int double_q, int32_t *greedy,
                               int32_t *next, float *filled_sum, double *scratch, void *stream) {
    if (!q_all || (!double_q && !q_tgt) || !filled || !greedy || !next || !filled_sum || !scratch) return XB_EINVAL;
    if (avail && avail_ld < A) return XB_EINVAL;
    int rc = qt_check(B, n, T, A);
    if (rc != XB_OK) return rc;
    qtran_select_kernel<<<qt_grid((int64_t)B * n * (T + 1)), 256, 0, (cudaStream_t)stream>>>(
        q_all, q_tgt, avail, avail_ld, filled, B, n, T, A, double_q, greedy, next, filled_sum, scratch);
    return xb_launch_status();
}

extern "C" int xb_qtran_encode_fwd(int mode, const float *state, int state_t0, const float *h,
                                   const float *agent_mask, const float *act_f, const int32_t *act_i, int act_T,
                                   const float *w1, const float *b1, const float *w2, const float *b2, int B, int n,
                                   int T, int S, int H, int A, float *x, float *pre, void *stream) {
    if (!state || !h || !agent_mask || !w1 || !b1 || !w2 || !b2 || !x) return XB_EINVAL;
    if (!act_f == !act_i || act_T < T || (state_t0 != 0 && state_t0 != 1)) return XB_EINVAL;
    int rc = qt_check_enc(mode, B, n, T, S, H, A);
    if (rc != XB_OK) return rc;
    const int D = H + A;
    const int smem = 4 * (2 * D * D + 4 * D + n * D);
    const int64_t R = (int64_t)B * T;
    const QtAct act{act_f, act_i, act_T};
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == XB_QTRAN_BASE) {
        if ((rc = qt_allow_smem(qtran_encode_fwd_kernel<XB_QTRAN_BASE>, smem)) != XB_OK) return rc;
        qtran_encode_fwd_kernel<XB_QTRAN_BASE><<<qt_persistent_grid(R, smem), QT_THREADS, smem, st>>>(
            state, state_t0, h, agent_mask, act, w1, b1, w2, b2, B, n, T, S, H, A, x, pre);
    } else {
        if ((rc = qt_allow_smem(qtran_encode_fwd_kernel<XB_QTRAN_ALT>, smem)) != XB_OK) return rc;
        qtran_encode_fwd_kernel<XB_QTRAN_ALT><<<qt_persistent_grid(R, smem), QT_THREADS, smem, st>>>(
            state, state_t0, h, agent_mask, act, w1, b1, w2, b2, B, n, T, S, H, A, x, pre);
    }
    return xb_launch_status();
}

// agent-rows per weight-gradient partial: 128, or more once there would be over QT_MAX_CHUNKS partials.  A function of
// R*n alone, so the reduction order (and the result's bits) does not depend on the device.
static int64_t qt_chunk_rows(int B, int n, int T) {
    const int64_t Rn = (int64_t)B * T * n;
    const int64_t c = (Rn + QT_MAX_CHUNKS - 1) / QT_MAX_CHUNKS;
    return c > QT_CHUNK ? c : QT_CHUNK;
}

static int64_t qt_chunks(int B, int n, int T) {
    const int64_t Rn = (int64_t)B * T * n, c = qt_chunk_rows(B, n, T);
    return (Rn + c - 1) / c;
}

extern "C" int64_t xb_qtran_encode_bwd_work(int B, int n, int T, int H, int A) {
    if (B <= 0 || n <= 0 || T <= 0 || H <= 0 || A <= 0) return 0;
    const int64_t D = H + A;
    return 2 * (int64_t)B * T * n * D + qt_chunks(B, n, T) * (2 * D * D + 2 * D);
}

extern "C" int xb_qtran_encode_bwd(int mode, const float *dx, const float *h, const float *agent_mask,
                                   const float *act_f, const int32_t *act_i, int act_T, const float *w1,
                                   const float *w2, const float *pre, int B, int n, int T, int S, int H, int A,
                                   float *dh, float *dw1, float *db1, float *dw2, float *db2, float *work,
                                   int64_t work_floats, void *stream) {
    if (!dx || !h || !agent_mask || !w1 || !w2 || !pre || !dh || !dw1 || !db1 || !dw2 || !db2 || !work)
        return XB_EINVAL;
    if (!act_f == !act_i || act_T < T) return XB_EINVAL;
    int rc = qt_check_enc(mode, B, n, T, S, H, A);
    if (rc != XB_OK) return rc;
    if (work_floats < xb_qtran_encode_bwd_work(B, n, T, H, A)) return XB_EINVAL;
    const int D = H + A;
    const int64_t R = (int64_t)B * T, Rn = R * n, nc = qt_chunks(B, n, T);
    float *GE = work, *DZ = work + Rn * D, *partial = DZ + Rn * D;
    const QtAct act{act_f, act_i, act_T};
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == XB_QTRAN_BASE) {
        const int smem = 4 * (2 * D * D + 3 * D);
        if ((rc = qt_allow_smem(qtran_encode_bwd_rows_kernel<XB_QTRAN_BASE>, smem)) != XB_OK) return rc;
        qtran_encode_bwd_rows_kernel<XB_QTRAN_BASE><<<qt_persistent_grid(R, smem), QT_THREADS, smem, st>>>(
            dx, S + D, agent_mask, w1, w2, pre, B, n, T, S, H, A, dh, GE, DZ);
    } else {
        const int smem = 4 * (2 * D * D + (n + 2) * D);
        if ((rc = qt_allow_smem(qtran_encode_bwd_rows_kernel<XB_QTRAN_ALT>, smem)) != XB_OK) return rc;
        qtran_encode_bwd_rows_kernel<XB_QTRAN_ALT><<<qt_persistent_grid(R, smem), QT_THREADS, smem, st>>>(
            dx, S + D + n, agent_mask, w1, w2, pre, B, n, T, S, H, A, dh, GE, DZ);
    }
    if ((rc = xb_launch_status()) != XB_OK) return rc;
    const dim3 wg((unsigned)nc, (unsigned)((D + QT_PTILE - 1) / QT_PTILE));
    qtran_encode_wgrad_kernel<<<wg, QT_WG_THREADS, 0, st>>>(h, agent_mask, act, pre, GE, DZ, B, n, T, H, A,
                                                             qt_chunk_rows(B, n, T), partial);
    if ((rc = xb_launch_status()) != XB_OK) return rc;
    const int NP = 2 * D * D + 2 * D;
    qtran_encode_wsum_kernel<<<(NP + 255) / 256, 256, 0, st>>>(partial, (int)nc, D, dw1, db1, dw2, db2);
    return xb_launch_status();
}

extern "C" int xb_qtran_loss_fwd_bwd(int mode, const float *q_all, const float *actions, const int32_t *greedy,
                                     const int32_t *next, const float *agent_mask, const float *filled,
                                     const float *rewards, const float *terminals, const float *qjt,
                                     const float *qjt_greedy, const float *qjt_next, const float *v,
                                     const float *filled_sum, int B, int n, int T, int A, float gamma,
                                     float lambda_opt, float lambda_nopt, int64_t rows_total, float *dqjt, float *dv,
                                     float *dq_all, float *stats, double *scratch, void *stream) {
    if (mode != XB_QTRAN_BASE && mode != XB_QTRAN_ALT) return XB_EINVAL;
    if (!q_all || !actions || !greedy || !next || !agent_mask || !filled || !rewards || !terminals || !qjt ||
        !qjt_greedy || !qjt_next || !v || !filled_sum || !dqjt || !dv || !dq_all || !stats || !scratch)
        return XB_EINVAL;
    int rc = qt_check(B, n, T, A);
    if (rc != XB_OK) return rc;
    const int64_t R = (int64_t)B * T;
    if (rows_total < R) return XB_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == XB_QTRAN_BASE)
        qtran_loss_kernel<XB_QTRAN_BASE><<<qt_grid(R), 256, 0, st>>>(
            q_all, actions, greedy, next, agent_mask, filled, rewards, terminals, qjt, qjt_greedy, qjt_next, v,
            filled_sum, B, n, T, A, gamma, lambda_opt, lambda_nopt, rows_total, dqjt, dv, dq_all, stats, scratch);
    else
        qtran_loss_kernel<XB_QTRAN_ALT><<<qt_grid(R), 256, 0, st>>>(
            q_all, actions, greedy, next, agent_mask, filled, rewards, terminals, qjt, qjt_greedy, qjt_next, v,
            filled_sum, B, n, T, A, gamma, lambda_opt, lambda_nopt, rows_total, dqjt, dv, dq_all, stats, scratch);
    return xb_launch_status();
}

// =====================================================================================================
// K13L  LSTM sequence kernels (the recurrence of a one-layer torch.nn.LSTM, gate order i, f, g, o)
// =====================================================================================================
// The same shape as K13 (gru.cu): one CTA walks all T steps of a slab of K13L_NS independent sequences, the slab's h
// and c live in shared memory between steps, and the only global traffic per step is xg[., t, :] in and y[., t, :]
// (+ the saved gates) out.  xb_lstm_seq_bwd walks the same slabs in reverse.  The time-independent GEMMs (input
// projection, dx, dW_ih, dW_hh) stay cuBLAS through torch.
//
// W_hh residency.  fp32 W_hh is 4H*H*4 B = 256 KB at H = 128, more than one CTA's 227 KB of shared memory, so each
// thread keeps the first K13L_KR = 32 entries of its k-range (forward: gate column j, k < 32; backward: the (gate, k)
// pair, jj < 32) in registers and the rest (k in [32, H)) sits in shared memory: 4 * 96 * 128 * 4 B = 192 KB at
// H = 128.  Register entries past H are zero and the slab's h / dgates buffers are zero-padded to max(H, 32), so a small
// H runs the same instruction stream with padded lanes multiplying zeros.
//
// Every sequence runs the same instructions in the same order whichever slab slot it lands in, so its results are
// bit-identical from launch to launch and across S.  No atomics, no fast-math intrinsics: expf / tanhf are the
// accurate libdevice versions, and the dot products run k in increasing order.
#include "xb_common.cuh"

#define K13L_NS 4        // sequences per CTA
#define K13L_MAX_H 128
#define K13L_KR 32       // k-entries of each thread's W_hh column held in registers

__device__ __forceinline__ float k13l_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

static inline int k13l_pad4(int H) { return (H + 3) & ~3; }
static inline int k13l_hs(int H) { return k13l_pad4(H) > K13L_KR ? k13l_pad4(H) : K13L_KR; }    // padded h width
static inline int k13l_ks(int H) { return k13l_pad4(H) > K13L_KR ? k13l_pad4(H) - K13L_KR : 0; }  // smem k-rows
static inline int k13l_threads(int H) { return (4 * H + 31) / 32 * 32; }

// shared memory: ws[KS][4H] (ws[k - 32][j] = W_hh[j][k], rows k >= H zero), hs[NS][HS] (zero-padded),
// ga[NS][4H] (the step's activated gates), cs[NS][H]
static inline size_t k13l_fwd_smem(int H) {
    const size_t G = 4 * (size_t)H;
    return sizeof(float) * ((size_t)k13l_ks(H) * G + (size_t)K13L_NS * k13l_hs(H) + K13L_NS * G + (size_t)K13L_NS * H);
}
// shared memory: wb[4][KS][H] (wb[p][jj - 32][k] = W_hh[p*H + jj][k], rows jj >= H zero), dg[NS][4][HS] (zero-padded),
// part[NS][4][H], dcs[NS][H]
static inline size_t k13l_bwd_smem(int H) {
    return sizeof(float) * ((size_t)4 * k13l_ks(H) * H + (size_t)K13L_NS * 4 * k13l_hs(H) + (size_t)K13L_NS * 4 * H +
                            (size_t)K13L_NS * H);
}

__global__ void __launch_bounds__(4 * K13L_MAX_H, 1)
    lstm_seq_fwd_kernel(const float *__restrict__ xg, const float *__restrict__ w_hh, const float *__restrict__ b_hh,
                        const float *__restrict__ h0, const float *__restrict__ c0, int64_t S, int T, int H,
                        float *__restrict__ y, float *__restrict__ hT, float *__restrict__ cT,
                        float *__restrict__ gates) {
    extern __shared__ __align__(16) float sm[];
    const int G = 4 * H, HP = (H + 3) & ~3;
    const int HS = HP > K13L_KR ? HP : K13L_KR, KS = HS - K13L_KR;
    float *ws = sm;
    float *hs = ws + KS * G;  // KS is a multiple of 4: float4-aligned
    float *ga = hs + K13L_NS * HS;
    float *cs = ga + K13L_NS * G;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int64_t s0 = (int64_t)blockIdx.x * K13L_NS;
    for (int i = tid; i < KS * G; i += nt) {
        const int k = K13L_KR + i / G, j = i % G;
        ws[i] = k < H ? w_hh[(int64_t)j * H + k] : 0.f;
    }
    for (int i = tid; i < K13L_NS * HS; i += nt) {
        const int s = i / HS, u = i - s * HS;
        const int64_t q = s0 + s;
        hs[i] = (h0 && u < H && q < S) ? h0[q * H + u] : 0.f;
    }
    for (int i = tid; i < K13L_NS * H; i += nt) {
        const int s = i / H, u = i - s * H;
        const int64_t q = s0 + s;
        cs[i] = (c0 && q < S) ? c0[q * H + u] : 0.f;
    }
    float wr[K13L_KR];
#pragma unroll
    for (int k = 0; k < K13L_KR; ++k) wr[k] = (tid < G && k < H) ? w_hh[(int64_t)tid * H + k] : 0.f;
    const float bj = tid < G ? b_hh[tid] : 0.f;
    const bool tanh_gate = tid >= 2 * H && tid < 3 * H;
    __syncthreads();
    for (int t = 0; t < T; ++t) {
        // pre[s][j] = xg[s, t, j] + (W_hh[j] . h_s + b_hh[j]), one gate column j per thread, k in increasing order
        if (tid < G) {
            float acc[K13L_NS];
#pragma unroll
            for (int s = 0; s < K13L_NS; ++s) acc[s] = 0.f;
#pragma unroll
            for (int k = 0; k < K13L_KR; k += 4) {
#pragma unroll
                for (int s = 0; s < K13L_NS; ++s) {
                    const float4 h = *reinterpret_cast<const float4 *>(hs + s * HS + k);
                    acc[s] = fmaf(wr[k], h.x, acc[s]);
                    acc[s] = fmaf(wr[k + 1], h.y, acc[s]);
                    acc[s] = fmaf(wr[k + 2], h.z, acc[s]);
                    acc[s] = fmaf(wr[k + 3], h.w, acc[s]);
                }
            }
            for (int k = K13L_KR; k < HS; k += 4) {
                const float *w = ws + (k - K13L_KR) * G + tid;
                const float w0 = w[0], w1 = w[G], w2 = w[2 * G], w3 = w[3 * G];
#pragma unroll
                for (int s = 0; s < K13L_NS; ++s) {
                    const float4 h = *reinterpret_cast<const float4 *>(hs + s * HS + k);
                    acc[s] = fmaf(w0, h.x, acc[s]);
                    acc[s] = fmaf(w1, h.y, acc[s]);
                    acc[s] = fmaf(w2, h.z, acc[s]);
                    acc[s] = fmaf(w3, h.w, acc[s]);
                }
            }
#pragma unroll
            for (int s = 0; s < K13L_NS; ++s) {
                const int64_t q = s0 + s;
                if (q >= S) continue;
                const int64_t row = q * T + t;
                const float pre = xg[row * G + tid] + (acc[s] + bj);
                const float a = tanh_gate ? tanhf(pre) : k13l_sigmoid(pre);
                ga[s * G + tid] = a;
                if (gates) gates[row * 5 * H + tid] = a;
            }
        }
        __syncthreads();
        // c' = f * c + i * g, h' = o * tanh(c')
        for (int i = tid; i < K13L_NS * H; i += nt) {
            const int s = i / H, u = i - s * H;
            const int64_t q = s0 + s;
            if (q >= S) continue;
            const int64_t row = q * T + t;
            const float *g = ga + s * G;
            const float c = g[H + u] * cs[i] + g[u] * g[2 * H + u];
            const float h = g[3 * H + u] * tanhf(c);
            cs[i] = c;
            hs[s * HS + u] = h;
            y[row * H + u] = h;
            if (gates) gates[row * 5 * H + 4 * H + u] = c;
        }
        __syncthreads();
    }
    for (int i = tid; i < K13L_NS * H; i += nt) {
        const int s = i / H, u = i - s * H;
        const int64_t q = s0 + s;
        if (q < S) {
            hT[q * H + u] = hs[s * HS + u];
            cT[q * H + u] = cs[i];
        }
    }
}

__global__ void __launch_bounds__(4 * K13L_MAX_H, 1)
    lstm_seq_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ dhT, const float *__restrict__ dcT,
                        const float *__restrict__ w_hh, const float *__restrict__ gates, const float *__restrict__ c0,
                        int64_t S, int T, int H, float *__restrict__ dxg, float *__restrict__ dh0,
                        float *__restrict__ dc0) {
    extern __shared__ __align__(16) float sm[];
    const int G = 4 * H, HP = (H + 3) & ~3;
    const int HS = HP > K13L_KR ? HP : K13L_KR, KS = HS - K13L_KR;
    float *wb = sm;
    float *dg = wb + 4 * KS * H;  // float4-aligned
    float *part = dg + K13L_NS * 4 * HS;
    float *dcs = part + K13L_NS * 4 * H;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int64_t s0 = (int64_t)blockIdx.x * K13L_NS;
    for (int i = tid; i < 4 * KS * H; i += nt) {
        const int pj = i / H, k = i - pj * H, p = pj / KS, jj = K13L_KR + pj - p * KS;
        wb[i] = jj < H ? w_hh[(int64_t)(p * H + jj) * H + k] : 0.f;
    }
    for (int i = tid; i < K13L_NS * 4 * HS; i += nt) dg[i] = 0.f;
    // part[s][0] starts as dhT so that dh = part0 + part1 + part2 + part3 + dy holds at t = T - 1 too
    for (int i = tid; i < K13L_NS * 4 * H; i += nt) {
        const int s = i / (4 * H), r = i - s * 4 * H;
        const int64_t q = s0 + s;
        part[i] = (dhT && r < H && q < S) ? dhT[q * H + r] : 0.f;
    }
    for (int i = tid; i < K13L_NS * H; i += nt) {
        const int s = i / H, u = i - s * H;
        const int64_t q = s0 + s;
        dcs[i] = (dcT && q < S) ? dcT[q * H + u] : 0.f;
    }
    const int p = tid / H, kk = tid - p * H;   // this thread's (gate, k) pair in W_hh^T dgates
    float wr[K13L_KR];
#pragma unroll
    for (int jj = 0; jj < K13L_KR; ++jj) wr[jj] = (tid < G && jj < H) ? w_hh[(int64_t)(p * H + jj) * H + kk] : 0.f;
    __syncthreads();
    for (int t = T - 1; t >= 0; --t) {
        // elementwise: dh_t = W_hh^T dgates_{t+1} + dy_t, dc_t = dc_{t+1} f_{t+1} + dh_t o_t (1 - tanh^2 c_t), then the
        // gate gradients of step t
        for (int i = tid; i < K13L_NS * H; i += nt) {
            const int s = i / H, u = i - s * H;
            const int64_t q = s0 + s;
            if (q >= S) continue;
            const int64_t row = q * T + t;
            const float *pp = part + s * 4 * H;
            const float dh = pp[u] + pp[H + u] + pp[2 * H + u] + pp[3 * H + u] + dy[row * H + u];
            const float *gt = gates + row * 5 * H;
            const float ig = gt[u], fg = gt[H + u], gg = gt[2 * H + u], og = gt[3 * H + u], c = gt[4 * H + u];
            const float cp = t > 0 ? gates[(row - 1) * 5 * H + 4 * H + u] : (c0 ? c0[q * H + u] : 0.f);
            const float tc = tanhf(c);
            const float dc = dcs[i] + dh * og * (1.f - tc * tc);
            const float di = dc * gg * (ig * (1.f - ig));
            const float df = dc * cp * (fg * (1.f - fg));
            const float dgg = dc * ig * (1.f - gg * gg);
            const float dO = dh * tc * (og * (1.f - og));
            float *dx = dxg + row * G;
            dx[u] = di;
            dx[H + u] = df;
            dx[2 * H + u] = dgg;
            dx[3 * H + u] = dO;
            float *d = dg + s * 4 * HS;
            d[u] = di;
            d[HS + u] = df;
            d[2 * HS + u] = dgg;
            d[3 * HS + u] = dO;
            dcs[i] = dc * fg;
        }
        __syncthreads();
        // part[s][p][k] = sum_{jj < H} W_hh[p*H + jj][k] * dgates_s[p*H + jj], jj in increasing order
        if (tid < G) {
            float acc[K13L_NS];
#pragma unroll
            for (int s = 0; s < K13L_NS; ++s) acc[s] = 0.f;
#pragma unroll
            for (int jj = 0; jj < K13L_KR; jj += 4) {
#pragma unroll
                for (int s = 0; s < K13L_NS; ++s) {
                    const float4 d = *reinterpret_cast<const float4 *>(dg + (s * 4 + p) * HS + jj);
                    acc[s] = fmaf(wr[jj], d.x, acc[s]);
                    acc[s] = fmaf(wr[jj + 1], d.y, acc[s]);
                    acc[s] = fmaf(wr[jj + 2], d.z, acc[s]);
                    acc[s] = fmaf(wr[jj + 3], d.w, acc[s]);
                }
            }
            const float *w = wb + p * KS * H + kk;
            for (int jj = K13L_KR; jj < HS; jj += 4) {
                const float *wj = w + (jj - K13L_KR) * H;
                const float w0 = wj[0], w1 = wj[H], w2 = wj[2 * H], w3 = wj[3 * H];
#pragma unroll
                for (int s = 0; s < K13L_NS; ++s) {
                    const float4 d = *reinterpret_cast<const float4 *>(dg + (s * 4 + p) * HS + jj);
                    acc[s] = fmaf(w0, d.x, acc[s]);
                    acc[s] = fmaf(w1, d.y, acc[s]);
                    acc[s] = fmaf(w2, d.z, acc[s]);
                    acc[s] = fmaf(w3, d.w, acc[s]);
                }
            }
#pragma unroll
            for (int s = 0; s < K13L_NS; ++s) part[(s * 4 + p) * H + kk] = acc[s];
        }
        __syncthreads();
    }
    for (int i = tid; i < K13L_NS * H; i += nt) {
        const int s = i / H, u = i - s * H;
        const int64_t q = s0 + s;
        if (q >= S) continue;
        const float *pp = part + s * 4 * H;
        if (dh0) dh0[q * H + u] = pp[u] + pp[H + u] + pp[2 * H + u] + pp[3 * H + u];
        if (dc0) dc0[q * H + u] = dcs[i];
    }
}

static inline bool k13l_shape_ok(int64_t S, int T, int H) {
    return S >= 1 && T >= 1 && H >= 1 && H <= K13L_MAX_H && (S + K13L_NS - 1) / K13L_NS <= 0x7fffffff;
}

extern "C" int xb_lstm_seq_fwd(const float *xg, const float *w_hh, const float *b_hh, const float *h0, const float *c0,
                               int64_t S, int T, int H, float *y, float *hT, float *cT, float *gates, void *stream) {
    if (!xg || !w_hh || !b_hh || !y || !hT || !cT) return XB_EINVAL;
    if (!k13l_shape_ok(S, T, H)) return XB_EINVAL;
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(lstm_seq_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)k13l_fwd_smem(K13L_MAX_H));
        attr = true;
    }
    const int grid = (int)((S + K13L_NS - 1) / K13L_NS);
    lstm_seq_fwd_kernel<<<grid, k13l_threads(H), k13l_fwd_smem(H), (cudaStream_t)stream>>>(xg, w_hh, b_hh, h0, c0, S,
                                                                                          T, H, y, hT, cT, gates);
    return xb_launch_status();
}

extern "C" int xb_lstm_seq_bwd(const float *dy, const float *dhT, const float *dcT, const float *w_hh,
                               const float *gates, const float *c0, int64_t S, int T, int H, float *dxg, float *dh0,
                               float *dc0, void *stream) {
    if (!dy || !w_hh || !gates || !dxg) return XB_EINVAL;
    if (!k13l_shape_ok(S, T, H)) return XB_EINVAL;
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(lstm_seq_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)k13l_bwd_smem(K13L_MAX_H));
        attr = true;
    }
    const int grid = (int)((S + K13L_NS - 1) / K13L_NS);
    lstm_seq_bwd_kernel<<<grid, k13l_threads(H), k13l_bwd_smem(H), (cudaStream_t)stream>>>(dy, dhT, dcT, w_hh, gates,
                                                                                          c0, S, T, H, dxg, dh0, dc0);
    return xb_launch_status();
}

// =====================================================================================================
// K13  GRU sequence kernels (the recurrence of a one-layer torch.nn.GRU, gate order r, z, n)
// =====================================================================================================
// xb_gru_seq_fwd walks all T steps of a slab of K13_NS independent sequences in one launch: W_hh stays resident in
// shared memory, the hidden states of the slab live in shared memory between steps, and the only global traffic per
// step is the projected input xg[., t, :] in and y[., t, :] (+ the saved gates) out.  xb_gru_seq_bwd walks the same
// slabs in reverse.  The time-independent GEMMs (input projection, dx, dW_ih, dW_hh) stay cuBLAS through torch.
//
// Every sequence runs the same instructions in the same order whichever slab slot it lands in (the padded lanes of
// a slab multiply zeros into nothing), so its results are bit-identical from launch to launch and across S.  No
// atomics, no fast-math intrinsics: expf / tanhf are the accurate libdevice versions.
#include "xb_common.cuh"

#define K13_NS 4        // sequences per CTA
#define K13_MAX_H 64

__device__ __forceinline__ float k13_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

static inline int k13_pad4(int H) { return (H + 3) & ~3; }
static inline int k13_threads(int H) { return (3 * H + 31) / 32 * 32; }

// shared memory: wt[HP][3H] (wt[k][j] = W_hh[j][k], rows k >= H zero), hs[NS][HP] (zero-padded), gh[NS][3H]
static inline size_t k13_fwd_smem(int H) {
    const int HP = k13_pad4(H);
    return sizeof(float) * ((size_t)HP * 3 * H + (size_t)K13_NS * HP + (size_t)K13_NS * 3 * H);
}
// shared memory: wb[3][HP][H] (wb[p][jj][k] = W_hh[p*H + jj][k], rows jj >= H zero), dg[NS][3][HP] (zero-padded),
// part[NS][3][H], dhz[NS][H]
static inline size_t k13_bwd_smem(int H) {
    const int HP = k13_pad4(H);
    return sizeof(float) * ((size_t)3 * HP * H + (size_t)K13_NS * 3 * HP + (size_t)K13_NS * 3 * H + (size_t)K13_NS * H);
}

__global__ void __launch_bounds__(192) gru_seq_fwd_kernel(const float *__restrict__ xg, const float *__restrict__ w_hh,
                                                          const float *__restrict__ b_hh, const float *__restrict__ h0,
                                                          int64_t S, int T, int H, float *__restrict__ y,
                                                          float *__restrict__ hT, float *__restrict__ gates) {
    extern __shared__ __align__(16) float sm[];
    const int G = 3 * H, HP = (H + 3) & ~3;
    float *wt = sm;
    float *hs = wt + HP * G;  // HP * G is a multiple of 4: float4-aligned
    float *gh = hs + K13_NS * HP;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int64_t s0 = (int64_t)blockIdx.x * K13_NS;
    for (int i = tid; i < HP * G; i += nt) {
        const int k = i / G, j = i - k * G;
        wt[i] = k < H ? w_hh[(int64_t)j * H + k] : 0.f;
    }
    for (int i = tid; i < K13_NS * HP; i += nt) {
        const int s = i / HP, u = i - s * HP;
        const int64_t q = s0 + s;
        hs[i] = (h0 && u < H && q < S) ? h0[q * H + u] : 0.f;
    }
    const float bj = tid < G ? b_hh[tid] : 0.f;
    __syncthreads();
    for (int t = 0; t < T; ++t) {
        // gh[s][j] = W_hh[j] . h_s + b_hh[j], one column j per thread, k in increasing order
        if (tid < G) {
            float acc[K13_NS];
#pragma unroll
            for (int s = 0; s < K13_NS; ++s) acc[s] = 0.f;
            for (int k = 0; k < HP; k += 4) {
                const float w0 = wt[k * G + tid], w1 = wt[(k + 1) * G + tid];
                const float w2 = wt[(k + 2) * G + tid], w3 = wt[(k + 3) * G + tid];
#pragma unroll
                for (int s = 0; s < K13_NS; ++s) {
                    const float4 h = *reinterpret_cast<const float4 *>(hs + s * HP + k);
                    acc[s] = fmaf(w0, h.x, acc[s]);
                    acc[s] = fmaf(w1, h.y, acc[s]);
                    acc[s] = fmaf(w2, h.z, acc[s]);
                    acc[s] = fmaf(w3, h.w, acc[s]);
                }
            }
#pragma unroll
            for (int s = 0; s < K13_NS; ++s) gh[s * G + tid] = acc[s] + bj;
        }
        __syncthreads();
        for (int i = tid; i < K13_NS * H; i += nt) {
            const int s = i / H, u = i - s * H;
            const int64_t q = s0 + s;
            if (q >= S) continue;
            const int64_t row = q * T + t;
            const float *x = xg + row * G;
            const float *g = gh + s * G;
            const float r = k13_sigmoid(x[u] + g[u]);
            const float z = k13_sigmoid(x[H + u] + g[H + u]);
            const float hn = g[2 * H + u];
            const float n = tanhf(x[2 * H + u] + r * hn);
            const float h = (1.f - z) * n + z * hs[s * HP + u];
            hs[s * HP + u] = h;
            y[row * H + u] = h;
            if (gates) {
                float *gt = gates + row * 4 * H;
                gt[u] = r;
                gt[H + u] = z;
                gt[2 * H + u] = n;
                gt[3 * H + u] = hn;
            }
        }
        __syncthreads();
    }
    for (int i = tid; i < K13_NS * H; i += nt) {
        const int s = i / H, u = i - s * H;
        const int64_t q = s0 + s;
        if (q < S) hT[q * H + u] = hs[s * HP + u];
    }
}

__global__ void __launch_bounds__(192) gru_seq_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ dhT,
                                                          const float *__restrict__ w_hh,
                                                          const float *__restrict__ gates, const float *__restrict__ y,
                                                          const float *__restrict__ h0, int64_t S, int T, int H,
                                                          float *__restrict__ dxg, float *__restrict__ dgh,
                                                          float *__restrict__ dh0) {
    extern __shared__ __align__(16) float sm[];
    const int G = 3 * H, HP = (H + 3) & ~3;
    float *wb = sm;
    float *dg = wb + 3 * HP * H;  // float4-aligned
    float *part = dg + K13_NS * 3 * HP;
    float *dhz = part + K13_NS * 3 * H;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int64_t s0 = (int64_t)blockIdx.x * K13_NS;
    for (int i = tid; i < 3 * HP * H; i += nt) {
        const int pj = i / H, k = i - pj * H, p = pj / HP, jj = pj - p * HP;
        wb[i] = jj < H ? w_hh[(int64_t)(p * H + jj) * H + k] : 0.f;
    }
    for (int i = tid; i < K13_NS * 3 * HP; i += nt) dg[i] = 0.f;
    for (int i = tid; i < K13_NS * 3 * H; i += nt) part[i] = 0.f;
    for (int i = tid; i < K13_NS * H; i += nt) {
        const int s = i / H, u = i - s * H;
        const int64_t q = s0 + s;
        dhz[i] = (dhT && q < S) ? dhT[q * H + u] : 0.f;
    }
    __syncthreads();
    for (int t = T - 1; t >= 0; --t) {
        // elementwise: dh_t = (dh_{t+1} z_{t+1} + W_hh^T dgh_{t+1}) + dy_t, then the gate gradients of step t
        for (int i = tid; i < K13_NS * H; i += nt) {
            const int s = i / H, u = i - s * H;
            const int64_t q = s0 + s;
            if (q >= S) continue;
            const int64_t row = q * T + t;
            const float *pp = part + s * 3 * H;
            const float dh = dhz[i] + pp[u] + pp[H + u] + pp[2 * H + u] + dy[row * H + u];
            const float *gt = gates + row * 4 * H;
            const float r = gt[u], z = gt[H + u], n = gt[2 * H + u], hn = gt[3 * H + u];
            const float hp = t > 0 ? y[(row - 1) * H + u] : (h0 ? h0[q * H + u] : 0.f);
            const float dnp = dh * (1.f - z) * (1.f - n * n);  // d(pre-tanh of n)
            const float dzp = dh * (hp - n) * (z * (1.f - z));
            const float drp = dnp * hn * (r * (1.f - r));
            const float dnh = dnp * r;                         // d(W_hn h + b_hn)
            float *dx = dxg + row * G, *dgo = dgh + row * G;
            dx[u] = drp;
            dx[H + u] = dzp;
            dx[2 * H + u] = dnp;
            dgo[u] = drp;
            dgo[H + u] = dzp;
            dgo[2 * H + u] = dnh;
            float *d = dg + s * 3 * HP;
            d[u] = drp;
            d[HP + u] = dzp;
            d[2 * HP + u] = dnh;
            dhz[i] = dh * z;
        }
        __syncthreads();
        // part[s][p][k] = sum_{jj < H} W_hh[p*H + jj][k] * dgh_s[p*H + jj], jj in increasing order
        if (tid < G) {
            const int p = tid / H, k = tid - p * H;
            const float *w = wb + p * HP * H + k;
            float acc[K13_NS];
#pragma unroll
            for (int s = 0; s < K13_NS; ++s) acc[s] = 0.f;
            for (int jj = 0; jj < HP; jj += 4) {
                const float w0 = w[jj * H], w1 = w[(jj + 1) * H], w2 = w[(jj + 2) * H], w3 = w[(jj + 3) * H];
#pragma unroll
                for (int s = 0; s < K13_NS; ++s) {
                    const float4 d = *reinterpret_cast<const float4 *>(dg + (s * 3 + p) * HP + jj);
                    acc[s] = fmaf(w0, d.x, acc[s]);
                    acc[s] = fmaf(w1, d.y, acc[s]);
                    acc[s] = fmaf(w2, d.z, acc[s]);
                    acc[s] = fmaf(w3, d.w, acc[s]);
                }
            }
#pragma unroll
            for (int s = 0; s < K13_NS; ++s) part[(s * 3 + p) * H + k] = acc[s];
        }
        __syncthreads();
    }
    if (dh0) {
        for (int i = tid; i < K13_NS * H; i += nt) {
            const int s = i / H, u = i - s * H;
            const int64_t q = s0 + s;
            const float *pp = part + s * 3 * H;
            if (q < S) dh0[q * H + u] = dhz[i] + pp[u] + pp[H + u] + pp[2 * H + u];
        }
    }
}

static inline bool k13_shape_ok(int64_t S, int T, int H) {
    return S >= 1 && T >= 1 && H >= 1 && H <= K13_MAX_H && (S + K13_NS - 1) / K13_NS <= 0x7fffffff;
}

extern "C" int xb_gru_seq_fwd(const float *xg, const float *w_hh, const float *b_hh, const float *h0, int64_t S, int T,
                              int H, float *y, float *hT, float *gates, void *stream) {
    if (!xg || !w_hh || !b_hh || !y || !hT) return XB_EINVAL;
    if (!k13_shape_ok(S, T, H)) return XB_EINVAL;
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(gru_seq_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)k13_fwd_smem(K13_MAX_H));
        attr = true;
    }
    const int grid = (int)((S + K13_NS - 1) / K13_NS);
    gru_seq_fwd_kernel<<<grid, k13_threads(H), k13_fwd_smem(H), (cudaStream_t)stream>>>(xg, w_hh, b_hh, h0, S, T, H,
                                                                                      y, hT, gates);
    return xb_launch_status();
}

extern "C" int xb_gru_seq_bwd(const float *dy, const float *dhT, const float *w_hh, const float *gates, const float *y,
                              const float *h0, int64_t S, int T, int H, float *dxg, float *dgh, float *dh0,
                              void *stream) {
    if (!dy || !w_hh || !gates || !y || !dxg || !dgh) return XB_EINVAL;
    if (!k13_shape_ok(S, T, H)) return XB_EINVAL;
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(gru_seq_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)k13_bwd_smem(K13_MAX_H));
        attr = true;
    }
    const int grid = (int)((S + K13_NS - 1) / K13_NS);
    gru_seq_bwd_kernel<<<grid, k13_threads(H), k13_bwd_smem(H), (cudaStream_t)stream>>>(dy, dhT, w_hh, gates, y, h0, S,
                                                                                      T, H, dxg, dgh, dh0);
    return xb_launch_status();
}

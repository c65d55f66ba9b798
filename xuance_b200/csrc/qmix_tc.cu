// K9-TC: the QMIX mixing network forward as ONE tensor-core kernel (wgmma, accumulators in registers).
//
//   Z      = X[rows x S] . W1cat^T[S x 128]              (first layers of hyper_w_1 | hyper_b_1 | hyper_w_2 | hyper_b_2)
//   W1raw  = relu(Z[:,  0: 32] + c) . Wb1^T [32 x n*32]  (second layer of hyper_w_1)
//   W2raw  = relu(Z[:, 64: 96] + c) . Wb2^T [32 x 32]    (second layer of hyper_w_2)
//   b2     = relu(Z[:, 96:128] + c) . wb2^T [32 x 1]     (second layer of hyper_b_2)
//   q_tot  = elu(q . |W1raw + c| + (Z[:,32:64] + c)) . |W2raw + c| + b2 + c         per row
// (xuance/torch/rl_models/heads/q_mix_head.py:52-95).  One CTA (two warpgroups) owns a tile of 128 rows, each
// warpgroup 64 of them (M = 64 per wgmma); the epilogues work on the accumulator fragments (tc_common.cuh).  All GEMM
// operands sit in shared memory in the K-major no-swizzle canonical
// layout (8-row x 16-byte core matrices), written by the threads themselves; the weights are staged once per CTA,
// the CTA then loops over its tiles (persistent grid = SM count).
//
// Numerics: the reference computes these layers in fp32.  The tensor pipe takes bf16 here, so every fp32 operand is
// split x = hi + lo (two bf16 values, |x - hi - lo| <= 2^-16 |x|) and each product is the sum of the three MMAs
// hi.hi + hi.lo + lo.hi (lo.lo <= 2^-16 relative, the size of the split residual itself) accumulated in fp32: relative error ~1e-5 per layer (a plain bf16 or TF32
// pass would be ~4e-3 / ~5e-4).  tests/test_gpu_qmix.py pins it against the fp32 oracle.
#include "tc_common.cuh"

namespace {
using namespace xbtc;

constexpr int TC_ROWS = 128;   // M
constexpr int TC_HH = 32;      // hypernet hidden = mixing hidden = 32 (the shipped QMIX configs)
constexpr int TC_N1 = 128;     // 4 x 32 first-layer outputs
constexpr int TC_THREADS = 256;  // two warpgroups, 64 rows each

// stage a [rows x K] fp32 row-major matrix (leading dimension ld; global OR shared memory) as hi/lo bf16 canonical
// operands, zero padded; one thread-iteration = 8 consecutive k of one row (two 16-byte shared-memory stores);
// U units are loaded before the first is used; (r, k0) advance incrementally (no division in the loop)
__device__ __forceinline__ void stage_operand(const float *__restrict__ g, int rows_valid, int rows_total, int K, int ld,
                                              int KP, uint8_t *hi, uint8_t *lo) {
    const int upr = KP >> 3;  // units per row
    const int total = rows_total * upr;
    constexpr int U = 4;
    const int dr = blockDim.x / upr, dk = blockDim.x - dr * upr;   // unit index += blockDim.x  <=>  (r += dr, ku += dk)
    int r = threadIdx.x / upr, ku = threadIdx.x - r * upr;
    for (int e0 = threadIdx.x; e0 < total; e0 += blockDim.x * U) {
        float x[U][8];
        int rr[U], kk[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            rr[u] = r, kk[u] = ku << 3;
            const float *src = g + (int64_t)r * ld + kk[u];
            const bool in = (e0 + u * (int)blockDim.x) < total && r < rows_valid;
#pragma unroll
            for (int i = 0; i < 8; ++i) x[u][i] = (in && kk[u] + i < K) ? src[i] : 0.f;
            r += dr, ku += dk;
            if (ku >= upr) ku -= upr, ++r;
        }
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (e0 + u * (int)blockDim.x < total) store_unit(x[u], rr[u], kk[u], KP, hi, lo);
    }
}

struct TcParams {
    const float *states, *q;                 // [R,S], [R,n]
    const float *w_l1[4], *b_l1[4];          // first layers of hyper_w_1 | hyper_b_1 | hyper_w_2 | hyper_b_2: [32,S], [32]
    const float *wb1, *bias_wb1;             // [n*32,32], [n*32]
    const float *wb2, *bias_wb2;             // [32,32], [32]
    const float *wb2c, *bias_wb2c;           // [1,32], [1]
    float *q_tot;                            // [R]
    int64_t R;
    int S, n;
};

__global__ void __launch_bounds__(TC_THREADS, 1) qmix_mix_tc_kernel(TcParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t x_bar;
    __shared__ float s_bias1[TC_N1], s_bias_wb1[256], s_bias_wb2[TC_HH], s_bias_b2;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wg = warp >> 2;                                         // warpgroup: rows 64 wg .. 64 wg + 63 of a tile
    const int S = p.S, n = p.n, KP1 = (S + 15) & ~15, N2A = n * TC_HH;
    // ---- shared memory carve-up (every operand base 128-B aligned)
    const int szA1 = TC_ROWS * KP1 * 2, szB1 = TC_N1 * KP1 * 2, szA2 = TC_ROWS * TC_HH * 2;
    const int szB2a = N2A * TC_HH * 2, szB2b = TC_HH * TC_HH * 2, szB2c = 16 * TC_HH * 2;
    uint8_t *A1h = smem, *A1l = A1h + szA1, *B1h = A1l + szA1, *B1l = B1h + szB1;
    // the three GEMM2 A operands (relu of the hidden blocks) reuse the X operand region: it is dead once GEMM1 completed
    uint8_t *A2h[3], *A2l[3];
    for (int i = 0; i < 3; ++i) {
        A2h[i] = A1h + (size_t)i * 2 * szA2;
        A2l[i] = A2h[i] + szA2;
    }
    uint8_t *B2ah = B1l + szB1, *B2al = B2ah + szB2a, *B2bh = B2al + szB2a, *B2bl = B2bh + szB2b;
    uint8_t *B2ch = B2bl + szB2b, *B2cl = B2ch + szB2c;
    float *Xraw = reinterpret_cast<float *>(B2cl + szB2c);   // [128 x S] fp32: the NEXT tile, fetched by the TMA unit
    // ---- one-time setup: mbarrier, weights
    const int64_t n_tiles = (p.R + TC_ROWS - 1) / TC_ROWS;
    // a tile is one contiguous run of rows_valid*S*4 bytes; the bulk copy needs a multiple of 16 bytes
    auto tile_copy_bytes = [&](int64_t t) -> uint32_t {
        const int64_t rows = (p.R - t * TC_ROWS) < TC_ROWS ? (p.R - t * TC_ROWS) : TC_ROWS;
        return (uint32_t)(rows * S * 4);
    };
    if (tid == 0) {
        mbar_init(&x_bar, 1);
        mbar_fence_init();
        if ((int64_t)blockIdx.x < n_tiles && (tile_copy_bytes(blockIdx.x) & 15) == 0) {   // prefetch the first tile
            mbar_expect_tx(&x_bar, tile_copy_bytes(blockIdx.x));
            bulk_g2s(Xraw, p.states + (int64_t)blockIdx.x * TC_ROWS * S, tile_copy_bytes(blockIdx.x), &x_bar);
        }
    }
    for (int blk = 0; blk < 4; ++blk)   // rows 32*blk .. 32*blk+31 of the concatenated first-layer weight
        stage_operand(p.w_l1[blk], TC_HH, TC_HH, S, S, KP1, B1h + (size_t)blk * (TC_HH / 8) * (KP1 / 8) * 128,
                      B1l + (size_t)blk * (TC_HH / 8) * (KP1 / 8) * 128);
    stage_operand(p.wb1, N2A, N2A, TC_HH, TC_HH, TC_HH, B2ah, B2al);
    stage_operand(p.wb2, TC_HH, TC_HH, TC_HH, TC_HH, TC_HH, B2bh, B2bl);
    stage_operand(p.wb2c, 1, 16, TC_HH, TC_HH, TC_HH, B2ch, B2cl);
    for (int i = tid; i < TC_N1; i += blockDim.x) s_bias1[i] = p.b_l1[i >> 5][i & 31];
    for (int i = tid; i < N2A; i += blockDim.x) s_bias_wb1[i] = p.bias_wb1[i];
    if (tid < TC_HH) s_bias_wb2[tid] = p.bias_wb2[tid];
    if (tid == 0) s_bias_b2 = p.bias_wb2c[0];
    __syncthreads();
    uint32_t xphase = 0;
    // this thread's rows (tile-relative) and first column of every 8-column block of a fragment
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
    // A operands: this warpgroup's 64 rows; B operands: row offsets of 8-row groups (KP * 2 bytes per row)
    const uint32_t a1h = smem_u32(A1h) + (uint32_t)(64 * wg * KP1 * 2), a1l = smem_u32(A1l) + (uint32_t)(64 * wg * KP1 * 2);

    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t row0 = tile * TC_ROWS;
        const int rows_valid = (int)((p.R - row0) < TC_ROWS ? (p.R - row0) : TC_ROWS);
        // ---- the agent utilities of this thread's two rows (latency hidden behind the staging + first GEMM)
        float qv[2][8];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 8; ++i) qv[h][i] = (i < n && r0 + 8 * h < rows_valid) ? p.q[(row0 + r0 + 8 * h) * n + i] : 0.f;
        // ---- stage X tile (split to bf16 hi/lo) from the prefetched raw copy (or from global for an unaligned tail)
        if ((tile_copy_bytes(tile) & 15) == 0) {
            mbar_wait(&x_bar, xphase);
            xphase ^= 1;
            stage_operand(Xraw, rows_valid, TC_ROWS, S, S, KP1, A1h, A1l);
        } else {
            stage_operand(p.states + row0 * S, rows_valid, TC_ROWS, S, S, KP1, A1h, A1l);
        }
        fence_proxy_async();   // generic-proxy smem writes -> visible to the tensor core (async proxy)
        __syncthreads();       // the whole X tile is staged (and Xraw consumed) before GEMM1 and the next prefetch
        if (tid == 0) {
            // Xraw was consumed by every thread (barrier above): fetch the next tile while this one computes
            const int64_t nt = tile + gridDim.x;
            if (nt < n_tiles && (tile_copy_bytes(nt) & 15) == 0) {
                mbar_expect_tx(&x_bar, tile_copy_bytes(nt));
                bulk_g2s(Xraw, p.states + nt * TC_ROWS * S, tile_copy_bytes(nt), &x_bar);
            }
        }
        // ---- GEMM1: Z[64 x 128] per warpgroup, products (hi,hi) (hi,lo) (lo,hi); lo.lo <= 2^-16 relative is dropped
        float z[4][16];
        wgmma_fence();
        {
            const uint32_t as[2] = {a1h, a1l}, bs[2] = {smem_u32(B1h), smem_u32(B1l)};
            uint32_t acc = 0;
            for (int pa = 0; pa < 2; ++pa)
                for (int pb = 0; pb < 2 - pa; ++pb)
                    for (int ks = 0; ks < KP1 / 16; ++ks) {   // one MMA = K 16 = two core matrices = 256 B along K
                        const uint64_t da = make_desc(as[pa] + ks * 256, KP1);
                        wgmma_n64<0, 0>(z[0], z[1], da, make_desc(bs[pb] + ks * 256, KP1), acc);
                        wgmma_n64<0, 0>(z[2], z[3], da, make_desc(bs[pb] + 64 * KP1 * 2 + ks * 256, KP1), acc);
                        acc = 1;
                    }
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncthreads();       // both warpgroups are done reading A1: the A2 operands overwrite it
        // ---- layer-1 epilogue: relu(Z + bias) of the three hidden blocks -> GEMM2 A operands; b1v = Z[:, 32:64] + bias
        float b1v[16];
        {
            const int blocks[3] = {0, 2, 3};
#pragma unroll
            for (int gi = 0; gi < 3; ++gi)
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int c = 8 * i + cq, bc = 32 * blocks[gi] + c;
                        store_pair(fmaxf(z[blocks[gi]][4 * i + 2 * h] + s_bias1[bc], 0.f),
                                   fmaxf(z[blocks[gi]][4 * i + 2 * h + 1] + s_bias1[bc + 1], 0.f), r0 + 8 * h, c, TC_HH, A2h[gi],
                                   A2l[gi]);
                    }
#pragma unroll
            for (int j = 0; j < 16; ++j) b1v[j] = z[1][j] + s_bias1[32 + 8 * (j >> 2) + cq + (j & 1)];
        }
        fence_proxy_async();
        __syncthreads();
        // ---- GEMM2: W1raw (one 32-column block per agent), W2raw, b2
        float w1[8][16], w2[16], b2[8];
        wgmma_fence();
        {
            const uint32_t off = (uint32_t)(64 * wg * TC_HH * 2);
            uint32_t acc = 0;
            for (int pa = 0; pa < 2; ++pa)
                for (int pb = 0; pb < 2 - pa; ++pb) {
                    const uint32_t ba = smem_u32(pb ? B2al : B2ah), bb = smem_u32(pb ? B2bl : B2bh), bc = smem_u32(pb ? B2cl : B2ch);
#pragma unroll
                    for (int ks = 0; ks < TC_HH / 16; ++ks) {
                        const uint32_t a0 = smem_u32(pa ? A2l[0] : A2h[0]) + off + ks * 256;
                        const uint32_t a1 = smem_u32(pa ? A2l[1] : A2h[1]) + off + ks * 256;
                        const uint32_t a2 = smem_u32(pa ? A2l[2] : A2h[2]) + off + ks * 256;
#pragma unroll
                        for (int i = 0; i < 8; ++i)
                            if (i < n)
                                wgmma_n32<0, 0>(w1[i], make_desc(a0, TC_HH), make_desc(ba + i * TC_HH * TC_HH * 2 + ks * 256, TC_HH), acc);
                        wgmma_n32<0, 0>(w2, make_desc(a1, TC_HH), make_desc(bb + ks * 256, TC_HH), acc);
                        wgmma_n16<0, 0>(b2, make_desc(a2, TC_HH), make_desc(bc + ks * 256, TC_HH), acc);
                        acc = 1;
                    }
                }
        }
        wgmma_commit();
        wgmma_wait<0>();
        // each warpgroup waited for its own wgmmas only: the next tile's staging overwrites A1, which the A2 operands alias,
        // so no thread may get there before BOTH warpgroups' GEMM2 has read them
        __syncthreads();
        // ---- mixing epilogue (q_mix_head.py:81-94) on the fragments: this thread holds 8 of the 32 hidden columns of
        // its two rows; the row sums over the hidden units are finished across the 4 lanes that share a row
        float pre[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) pre[j] = b1v[j];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (i < n) {
#pragma unroll
                for (int j = 0; j < 16; ++j)
                    pre[j] += qv[(j >> 1) & 1][i] * fabsf(w1[i][j] + s_bias_wb1[i * TC_HH + 8 * (j >> 2) + cq + (j & 1)]);
            }
        }
        float y[2] = {0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float hv = pre[j] > 0.f ? pre[j] : (expf(pre[j]) - 1.f);
            y[(j >> 1) & 1] += hv * fabsf(w2[j] + s_bias_wb2[8 * (j >> 2) + cq + (j & 1)]);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            y[h] += __shfl_xor_sync(0xffffffffu, y[h], 1);
            y[h] += __shfl_xor_sync(0xffffffffu, y[h], 2);
        }
        // b2 is column 0 of its fragment: registers 0 (row r0) and 2 (row r0 + 8) of the lane with lane % 4 == 0
        if ((lane & 3) == 0) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (r0 + 8 * h < rows_valid) p.q_tot[row0 + r0 + 8 * h] = y[h] + b2[2 * h] + s_bias_b2;
        }
    }
}

}  // namespace

extern "C" int xb_qmix_mix_fused_fwd(const float *states, const float *q, const float *const *w_l1,
                                     const float *const *b_l1, const float *wb1, const float *bias_wb1,
                                     const float *wb2, const float *bias_wb2, const float *wb2c,
                                     const float *bias_wb2c, int64_t R, int S, int n, int H, int HH, float *q_tot,
                                     void *stream) {
    if (!states || !q || !w_l1 || !b_l1 || !wb1 || !bias_wb1 || !wb2 || !bias_wb2 || !wb2c || !bias_wb2c || !q_tot)
        return XB_EINVAL;
    for (int i = 0; i < 4; ++i)
        if (!w_l1[i] || !b_l1[i]) return XB_EINVAL;
    if (R <= 0 || S <= 0 || n <= 0) return XB_EINVAL;
    if (H != TC_HH || HH != TC_HH || n > 8 || S > 160) return XB_ERANGE;   // shapes of the shipped QMIX configs
    const int KP1 = (S + 15) & ~15;
    const size_t smem = (size_t)2 * TC_ROWS * KP1 * 2 + (size_t)2 * TC_N1 * KP1 * 2 + 2 * (size_t)n * TC_HH * TC_HH * 2 +
                        2 * TC_HH * TC_HH * 2 + 2 * 16 * TC_HH * 2 + (size_t)TC_ROWS * S * 4;
    if ((size_t)6 * TC_ROWS * TC_HH * 2 > (size_t)2 * TC_ROWS * KP1 * 2) return XB_ERANGE;   // A2 operands alias A1
    if (smem > 220 * 1024) return XB_ERANGE;
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(qmix_mix_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
        attr = true;
    }
    TcParams p{states, q, {w_l1[0], w_l1[1], w_l1[2], w_l1[3]}, {b_l1[0], b_l1[1], b_l1[2], b_l1[3]},
               wb1, bias_wb1, wb2, bias_wb2, wb2c, bias_wb2c, q_tot, R, S, n};
    int64_t tiles = (R + TC_ROWS - 1) / TC_ROWS;
    int grid = (int)(tiles < xb_sm_count() ? tiles : xb_sm_count());
    qmix_mix_tc_kernel<<<grid, TC_THREADS, smem, (cudaStream_t)stream>>>(p);
    return xb_launch_status();
}

// K12: gathered-operand GEMM on the Hopper tensor cores (wgmma, accumulators in registers) for the NatureCNN layers
// (cnn.py:45-50, 84-101) - forward, data gradient, weight gradient and bias gradient of the three convolutions and the hidden
// layer, the bulk of the fp32 PPO step that cuDNN's CUDA-core fp32 convolutions took (DESIGN.md sections 3, 3a, 7).
//
//   D[m, n] = sum_{t, c} in[b, y*sy + dy[t], x*sx + dx[t], c] * W[n, t*C + c]  (+ bias[n], ReLU)      conv_index.h
//
// Numerics: every fp32 operand travels as 1-3 bf16 planes (x = sum of its planes); the kept plane products are accumulated
// in fp32, one accumulator per order of magnitude, and added smallest first in the epilogue (see the kernel).
//
// Structure (one CTA per SM, persistent over work items = (128-row tile, column tile[, split]), 12 warps):
//   warps 8-11 producers : four ways to fill a stage, chosen per operand by the host entry point:
//                          * TMA tiles with the 128-byte swizzle for plain matrices (packed weights, output gradients, the
//                            Linear layer's inputs), all planes of an operand in one cp.async.bulk.tensor;
//                          * TMA boxes over padded-row activations (a_box: xb_gemm_box_tc / xb_wgrad_box_tc), rank-5 view
//                            {channel, pixel, row phase, row / stride, plane};
//                          * a RESIDENT activation tile (a_halo: xb_gemm_halo_tc) - one box per plane and M tile, taps are
//                            descriptor offsets, only the weights stream through the ring;
//                          * 16-byte cp.async gathers into the no-swizzle canonical layout (conv1's raw pixels): each of the
//                            128 threads plays producers pt and pt + 128 of the 256-thread mapping of conv_index.h,
//                            row-coalesced, zero-fill for padding taps, ASYNCHRONOUS arrival on the stage's full barrier
//                            (cp.async.mbarrier.arrive.noinc).
//                          One elected thread arms the barrier with the TMA byte count; no producer waits for a load.
//   warps 0-7  consumers : two warpgroups, rows 0-63 and 64-127 of the tile (M = 64 per wgmma).  Per K step of 16 and A plane
//                          pa, wgmmas of 64 / 32 columns multiply it with the first PB - pa B planes (adjacent in the stage =
//                          ONE operand of (PB - pa) * N rows) into the register accumulator blocks of groups pa .. PB-1; a
//                          stage is released when the wgmma group after it was issued has retired the one that read it.
//                          The epilogue runs on the fragments: accumulator groups added smallest first, bias + ReLU /
//                          ReLU-derivative mask, the rows written as fp32 and / or as the bf16 planes the next layer consumes
//                          (into its padded layout), and the column sums of the tile (the bias-gradient partials of the layer
//                          below).
#include <cstdlib>

#include <cuda.h>      // CUtensorMap + the cuTensorMapEncodeTiled prototype (resolved at run time through the runtime API)

#include "tc_common.cuh"
#include "conv_index.h"

namespace {
using namespace xbtc;

constexpr int KC = XB_CONV_KC, TILE_M = XB_CONV_TILE_M;
constexpr int CONS_WARPS = 8;                              // two consumer warpgroups
constexpr int PROD_THREADS = XB_CONV_PRODUCERS / 2;        // one producer warpgroup, two conv_index.h producers per thread
constexpr int THREADS = CONS_WARPS * 32 + PROD_THREADS;
constexpr int MAX_STAGES = 6;
constexpr int XB_HALO_MAX_CHUNKS = 16;
constexpr int XB_K12_MAX_DYN_SMEM = 208 * 1024;      // + ~18 KB static (barriers, bias, column sums, tap table) <= 227 KB

// Optional role timing (XB_K12_TIMING=1): clock64 cycles each role of CTA b spent inside its barrier waits, written at kernel
// exit to xb_k12_timing[b][..]: 0 consumer total, 1 consumer wait full (operands), 3 consumer wait a_full (halo tile),
// 4 producer total, 5 producer wait empty (ring), 6 producer wait a_empty (tools/k12_timing.py); the other slots are unused
__device__ unsigned long long xb_k12_timing[160][12];

struct ConvParams {
    // TMA descriptors of the operands that are plain matrices (bf16 planes as the outermost dimension): the B operand
    // (packed weights [N_total, K] forward, output gradient [sites, g_ld] in the weight gradient) and, for a Linear layer,
    // the A operand.  Gathered A operands (convolutions) keep the cp.async path.
    alignas(64) CUtensorMap tm_a;
    alignas(64) CUtensorMap tm_b;
    int a_tma, b_tma;
    // a_box: the A operand of a convolution fetched by TMA as ONE 4-D box per plane and chunk from an activation tensor
    // stored with padded rows, {channels, pixels, merged image-rows, planes}: a tile is box_h consecutive grid rows of box_w
    // sites; chunk kc reads the box at (box_c0[kc], box_w0[kc], tile_row0 * box_rs + box_r[kc]).  Output rows are decoded as
    // (merged row R = tile * box_h + r / box_w, x = r % box_w), image b = R / box_hp, y = R % box_hp, valid if
    // box_y0 <= y <= box_y1 (rows outside are the padding / garbage rows of the padded layout and are never written).
    int a_box, box_w, box_h, box_hp, box_y0, box_y1, box_rs, box_chunks;
    XbDiv box_div_w, box_div_hp;
    int16_t box_c0[16], box_w0[16], box_r[16];
    // a_halo: stride-1 gathers over a 64-channel padded-row tensor [planes][B*hp rows][W pixels][64] with the activation tile
    // RESIDENT in shared memory: the sites are the positions P of the haloed raster (row R, column hc: pixel hc + halo_w0,
    // halo_w columns per row), an M tile is 128 consecutive positions, and ONE box per plane of halo_rows rows x halo_w pixels
    // (OOB pixels / rows zero-filled) holds every input any tap of the tile reads; chunk kc of sub-item nt reads the 128
    // consecutive tile rows that start halo_shift[nt*halo_chunks + kc] = dr*halo_w + dc positions after the site's own - a
    // descriptor offset, not a new load.  Only the weights stream through the ring.  The n tiles of an M tile (stride phases
    // of a data gradient: own weights rows nt*N.., own output placement sub_oy0 / sub_ox0 and valid extent sub_y1 / sub_x1)
    // run back to back on the same tile.
    int a_halo, halo_w, halo_w0, halo_rows, halo_lo, halo_chunks, halo_same_cols;
    int64_t halo_positions;                // B * hp * halo_w
    XbDiv halo_div_w;
    int16_t halo_shift[XB_HALO_MAX_CHUNKS];
    int16_t sub_oy0[4], sub_ox0[4], sub_y1[4], sub_x1[4];
    XbConvGeom g;                          // g.N = columns per work item (the tile width N)
    const __nv_bfloat16 *in[3];            // A planes: [B, IH, IW, C]
    const __nv_bfloat16 *w[3];             // B planes.  forward: weight [N_total, K].  weight gradient: output gradient [P, w_ld]
    const float *bias;                     // [N_total] or null (forward)
    int mask_W, mask_x0;                   // box mode: the mask tensor's row width / pixel offset (its rows as the output's)
    int64_t mask_ld;                       // the mask tensor's channels per pixel and first channel (as out_ld / out_c0)
    int mask_c0;
    float *colsum;                         // forward, nullable: [work items of M][N total] column sums of the rows this
                                           // item wrote (after bias / ReLU / mask) - the next layer's bias-gradient partials
    const __nv_bfloat16 *mask;             // forward, nullable: result elements are zeroed where mask <= 0; same
                                           // addressing as the output (the ReLU derivative of a saved activation's hi plane)
    __nv_bfloat16 *out[3];                 // forward: p_out result planes (nullable)
    float *out_f32;                        // forward: nullable.  weight gradient: partials [splits, K, N_total]
    int64_t M;                             // sites B * OY * OX (GEMM rows forward, reduction length for the weight gradient)
    int relu, stages, p_out;
    uint32_t dyn_smem;                     // dynamic shared memory of the launch (0: stages * stage bytes)
    int timing;                            // XB_K12_TIMING: fill xb_k12_timing
    // forward: placement of site (b, y, x): row ((b*out_H + y*oys + oy0)*out_W + x*oxs + ox0) of an output matrix whose
    // rows are out_ld elements apart; work item (m tile, n tile nt) fills columns [out_c0 + nt*N, out_c0 + (nt+1)*N)
    int out_H, out_W, oys, oxs, oy0, ox0;
    int64_t out_ld;
    int out_c0;
    int n_tiles;                           // column tiles per row tile (N_total = n_tiles * N)
    int64_t w_ld;                          // weight gradient: elements between consecutive sites of the output gradient
    // weight gradient: sites are cut into `splits` runs of sites_per_split (a multiple of KC)
    int splits;
    int64_t sites_per_split;
};

// 16-byte cp.async with zero-fill.  CA = through L1 (sector sharing between the lanes of a request and reuse of the
// overlapping windows of the raw-pixel first layer); otherwise L2 only (better for the wider layers).
template <bool CA>
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, uint32_t src_bytes) {
    if (CA) asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
    else asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// TMA: one 3-D tile {c0 .. c0+box0, c1 .. c1+box1, all planes} -> shared memory, completion bytes on an mbarrier
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *tm, int c0, int c1, int c2, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
        : "memory");
}
// one box of a padded-row activation tensor viewed as {channels, pixels, row phase (row mod S), row / S, plane}: row `r` of
// the tensor is (phase r mod S, index r / S), so a convolution of stride S reads CONSECUTIVE indices of ONE phase - no
// traversal stride is needed (a 64-byte inner box under the 128-byte swizzle pads every pixel to a 128-byte row, so
// 32-channel tensors are described as 64-channel pixel pairs instead, see BoxNatureCNN)
__device__ __forceinline__ void tma_load_box(uint32_t dst, const CUtensorMap *tm, int c, int w, int row, int S, int plane,
                                             uint64_t *bar) {
    const int idx = S == 1 ? row : (row >= 0 ? row / S : -((-row + S - 1) / S));      // floor(row / S)
    const int ph = row - idx * S;
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
        ::"r"(dst), "l"(tm), "r"(c), "r"(w), "r"(ph), "r"(idx), "r"(plane), "r"(smem_u32(bar))
        : "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// x = hi + mid + lo, three bf16 values: 24 mantissa bits, |x - hi - mid - lo| <= 2^-24 |x|
__device__ __forceinline__ void split3_bf16(float x, __nv_bfloat16 &hi, __nv_bfloat16 &mid, __nv_bfloat16 &lo) {
    hi = __float2bfloat16_rn(x);
    const float r1 = x - __bfloat162float(hi);
    mid = __float2bfloat16_rn(r1);
    lo = __float2bfloat16_rn(r1 - __bfloat162float(mid));
}

// A plane x the first PB - pa B planes for one K step: the accumulator blocks pa*NC .. PB*NC-1 (32 columns each).  Block j
// reads B rows 32 (j - pa*NC) .. +31 of the stage: 4096 bytes per block in every operand layout the kernel uses (128 bytes
// per row or per MN index).  In-flight wgmmas are ordered on their accumulator registers only when they have the same shape
// and register set, so every block is always written by the same instruction form: pairs (2i, 2i+1) as one n64 wgmma when
// NC is even (then every plane's range starts at an even block), single n32 wgmmas when NC is odd.
template <int T, int PB, int NC, int PA_>
__device__ __forceinline__ void mma_plane(float (&acc)[PB * NC][16], uint64_t da, uint64_t db, uint32_t scale_d) {
    constexpr int J0 = PA_ * NC, J1 = PB * NC, STEP = NC % 2 == 0 ? 2 : 1;
#pragma unroll
    for (int j = J0; j < J1; j += STEP) {
        const uint64_t b = db + (uint64_t)(((j - J0) * 4096) >> 4);
        if (STEP == 2) wgmma_n64<T, T>(acc[j], acc[j + 1 < J1 ? j + 1 : j], da, b, scale_d);
        else wgmma_n32<T, T>(acc[j], da, b, scale_d);
    }
}

// WGRAD = false:  D[site, n]  = sum_k A[site, k] W[n, k]            work item = (128-site tile, n tile),        K-major operands
// WGRAD = true :  D[kcol, n]  = sum_site A[site, kcol] G[site, n]   work item = (128-kcol tile, n tile, split), MN-major operands
// PA / PB: bf16 planes of the A / B operand (x = sum of its planes, plane q = bf16 of the residual left by planes < q),
// PA <= PB.  NC: the tile width N = 32 NC.  The products kept are those whose plane indices sum to < PB; they are accumulated
// in PB SEPARATE float32 accumulators D_g, g = pa + pb, which the epilogue adds smallest first: the tensor core truncates
// (rounds toward zero) when it adds a product block into the accumulator, so keeping the 2^-8 / 2^-16 sized correction terms
// out of the hi.hi accumulator both shortens its chain of truncating additions by the number of products and keeps the
// corrections' own truncation error at 2^-8 / 2^-16 of an ulp of the result.  The B planes of a stage are adjacent in shared
// memory, so in the canonical layouts they ARE one operand of PB*N rows: the wgmmas of one A plane multiply it with the
// first (PB - pa) B planes and land in the accumulator columns of groups pa .. PB-1.
template <bool WGRAD, int PA, int PB, int NC>
__global__ void __launch_bounds__(THREADS, 1) conv_tc_kernel(const __grid_constant__ ConvParams p) {
    static_assert(PA >= 1 && PA <= PB && PB <= 3 && PB * NC <= 8, "plane counts / tile width");
    constexpr int N = 32 * NC;
    constexpr int TR = WGRAD ? 1 : 0;                 // both operands MN-major in the weight gradient
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t full_bar[MAX_STAGES], empty_bar[MAX_STAGES], a_full[2], a_empty[2];
    __shared__ float s_bias[N];
    __shared__ float s_colsum[CONS_WARPS][N];         // per consumer warp: column sums of its 16 rows (ConvParams.colsum)
    __shared__ XbUnit s_units[XB_CONV_MAX_UNITS];     // per 16-byte K unit: tap offsets + element offset (conv_index.h)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const XbConvGeom &g = p.g;
    const int K = g.T * g.C, S = p.stages;
    const uint32_t a_plane = xb_conv_a_plane_bytes(), w_plane = xb_conv_w_plane_bytes(N);
    const bool halo = !WGRAD && p.a_halo;
    const uint32_t halo_plane = halo ? (((uint32_t)(p.halo_rows * p.halo_w) * 128u + 1023u) & ~1023u) : 0u;   // one plane of a tile
    const uint32_t a_buf_bytes = PA * halo_plane, ring_off = 2u * a_buf_bytes;       // two resident A tiles, then the ring
    const uint32_t stage_bytes = (halo ? 0u : PA * a_plane) + PB * w_plane;
    const int box_rows = p.box_w * p.box_h;                  // a_box: rows of a tile that hold sites (<= 128)
    const int64_t m_tiles = WGRAD ? (K + TILE_M - 1) / TILE_M
                                  : halo ? (p.halo_positions + TILE_M - 1) / TILE_M
                                  : (p.a_box ? ((int64_t)g.B * p.box_hp + p.box_h - 1) / p.box_h : (p.M + TILE_M - 1) / TILE_M);
    const int64_t mn_tiles = m_tiles * p.n_tiles;
    // the persistent loop walks n_work outer items with n_inner sub-items each: (m tile, n tile[, split]) one by one, or in
    // halo mode M tiles with their n tiles back to back (they share the resident activation tile)
    const int64_t n_work = WGRAD ? mn_tiles * p.splits : (halo ? m_tiles : mn_tiles);
    const int n_inner = halo ? p.n_tiles : 1;
    // halo: first tensor row of the tile of M tile `t` (floor((128 t + halo_lo) / halo_w), the numerator kept positive)
    auto halo_row_lo = [&](int64_t t) -> int {
        const uint32_t num = (uint32_t)(t * TILE_M + p.halo_lo + 4 * p.halo_w);
        return (int)xb_div(num, p.halo_div_w) - 4;
    };
    // chunks of one work item
    auto chunks_of = [&](int64_t w) -> int {
        if (!WGRAD) return halo ? p.halo_chunks : (p.a_box ? p.box_chunks : K / KC);
        const int64_t sp = w / mn_tiles, s0 = sp * p.sites_per_split;
        const int64_t cnt = (p.M - s0) < p.sites_per_split ? (p.M - s0) : p.sites_per_split;
        // a_box: the reduction runs over merged grid rows (p.M of them), box_h rows = box_h * box_w <= 64 sites per chunk
        return p.a_box ? (int)((cnt + p.box_h - 1) / p.box_h) : (int)((cnt + KC - 1) / KC);
    };

    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            // one asynchronous arrival per producer thread (+ the expect_tx arrival of the thread that issues the TMA copies)
            mbar_init(&full_bar[s], halo ? 1 : PROD_THREADS + ((p.a_tma || p.b_tma) ? 1 : 0));
            mbar_init(&empty_bar[s], CONS_WARPS);
        }
        for (int a = 0; a < 2; ++a) {
            mbar_init(&a_full[a], 1);
            mbar_init(&a_empty[a], CONS_WARPS);
        }
        mbar_fence_init();
    }
    if (!p.a_box && !halo)
        for (int i = tid; i < K / 8; i += THREADS) s_units[i] = xb_unit(g, i);
    if (WGRAD && p.a_box) {
        // a chunk holds box_h * box_w <= 64 sites: the rows of each 64-site block that no box ever writes must read as zero
        const uint32_t total = (uint32_t)S * stage_bytes;
        for (uint32_t i = tid * 16u; i < total; i += THREADS * 16u) *reinterpret_cast<uint4 *>(smem + i) = make_uint4(0, 0, 0, 0);
        fence_proxy_async();
    }
    __syncthreads();
    const uint32_t smem_base = smem_u32(smem);
    unsigned long long t_wait[3] = {0, 0, 0};
    const unsigned long long t_begin = p.timing ? clock64() : 0ull;
    auto timed_wait = [&](uint64_t *bar, uint32_t parity, int slot) {
        if (p.timing) {
            const unsigned long long t0 = clock64();
            mbar_wait(bar, parity);
            t_wait[slot] += clock64() - t0;
        } else {
            mbar_wait(bar, parity);
        }
    };
    if ((p.a_tma || p.b_tma) && (smem_base & 1023u)) __trap();     // the 128-byte swizzle pattern repeats every 1024 B

    if (warp >= CONS_WARPS) {
        // ------------------------------------------------------------------ producers (128 threads)
        const int ptb = tid - CONS_WARPS * 32;
        uint32_t it = 0, tile_it = 0;
        if (!(halo && ptb != 0))                               // halo: both operands by TMA, one thread drives them
        for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x) {
          if (halo) {
              // the activation tile of this M tile: one box per plane into the buffer the tile before the last one used
              const uint32_t buf = tile_it & 1u;
              timed_wait(&a_empty[buf], ((tile_it >> 1) & 1u) ^ 1u, 1);
              mbar_expect_tx(&a_full[buf], (uint32_t)PA * (uint32_t)(p.halo_rows * p.halo_w) * 128u);
              const int r_lo = halo_row_lo(w);
#pragma unroll
              for (int q = 0; q < PA; ++q)
                  tma_load_box(smem_base + buf * a_buf_bytes + q * halo_plane, &p.tm_a, 0, p.halo_w0, r_lo, 1, q, &a_full[buf]);
              ++tile_it;
          }
          for (int sub = 0; sub < n_inner; ++sub) {
            const int n_chunks = chunks_of(w);
            const int64_t sp = WGRAD ? w / mn_tiles : 0;
            const int64_t rem = WGRAD ? w - sp * mn_tiles : w;
            const int64_t mt = halo ? w : rem / p.n_tiles;
            const int nt = halo ? sub : (int)(rem - mt * p.n_tiles);
            XbSite sites[4];                                   // forward: the four rows this thread feeds (both of its producers)
            if (!WGRAD && !p.a_tma && !halo) {
#pragma unroll
                for (int gi = 0; gi < 4; ++gi) sites[gi] = xb_site(g, mt * TILE_M + xb_fwd_row(ptb, gi), p.M);
            }
            const int64_t w_off = WGRAD ? 0 : (int64_t)nt * N * K;        // forward: first weight row of this n tile
            const int64_t site_end = WGRAD ? ((sp + 1) * p.sites_per_split < p.M ? (sp + 1) * p.sites_per_split : p.M) : 0;
            for (int kc = 0; kc < n_chunks; ++kc) {
                const int stage = (int)(it % (uint32_t)S);
                timed_wait(&empty_bar[stage], ((it / (uint32_t)S) & 1u) ^ 1u, 0);
                const uint32_t base = smem_base + ring_off + (uint32_t)stage * stage_bytes;
                const uint32_t wbase = base + (halo ? 0u : PA * a_plane);
                auto emit_a = [&](uint32_t dst_off, int64_t src) {       // src < 0: the 16 bytes are zero-filled
                    if (p.a_tma) return;
                    const uint32_t nbytes = src >= 0 ? 16u : 0u;
                    const int64_t o = src >= 0 ? src : 0;
#pragma unroll
                    for (int q = 0; q < PA; ++q) cp_async16<PA == 1>(base + q * a_plane + dst_off, p.in[q] + o, nbytes);
                };
                auto emit_w = [&](uint32_t dst_off, int64_t src) {
                    if (p.b_tma) return;
                    const uint32_t nbytes = src >= 0 ? 16u : 0u;
                    const int64_t o = src >= 0 ? src + w_off : 0;
#pragma unroll
                    for (int q = 0; q < PB; ++q) cp_async16<false>(wbase + q * w_plane + dst_off, p.w[q] + o, nbytes);
                };
                const int64_t site0 = sp * p.sites_per_split + (int64_t)kc * KC;     // weight gradient: first site of the chunk
                if (ptb == 0 && (p.a_tma || p.b_tma)) {
                    // plain-matrix operands: one elected thread arms the barrier with the byte count and issues the tile
                    // copies; every plane of an operand travels in ONE box (planes are the outermost tensor dimension)
                    uint32_t bytes = (p.a_tma ? PA * (p.a_box ? (uint32_t)box_rows * 128u : a_plane) : 0u) + (p.b_tma ? PB * w_plane : 0u);
                    if (p.a_box && WGRAD) {                 // blocks of this tile that exist (1 or 2) + the G box, box_rows sites each
                        const int nblk = ((int)mt * 2 + 1 < p.box_chunks) ? 2 : 1;
                        bytes = (uint32_t)(nblk * PA + PB) * (uint32_t)box_rows * 128u;
                    }
                    mbar_expect_tx(&full_bar[stage], bytes);
                    if (p.b_tma && !(p.a_box && WGRAD)) {
                        if (!WGRAD) tma_load_3d(wbase, &p.tm_b, kc * KC, nt * N, 0, &full_bar[stage]);          // W[n, k] rows
                        else tma_load_3d(wbase, &p.tm_b, nt * N, (int)site0, 0, &full_bar[stage]);               // G[site, n] rows
                    }
                    if (p.a_box && WGRAD) {
                        // weight gradient over padded-row tensors: the chunk is box_h grid rows of the site grid; the two
                        // 64-column blocks of the tile are the forward's K chunks 2*mt and 2*mt+1 (same box tables); G is a
                        // box of the padded output-gradient tensor.  (bytes: see the expect_tx above)
                        const int row0 = (int)(sp * p.sites_per_split) + kc * p.box_h;
                        for (int j = 0; j < 2; ++j) {
                            const int ci = (int)mt * 2 + j;
                            if (ci >= p.box_chunks) break;
#pragma unroll
                            for (int q = 0; q < PA; ++q)
                                tma_load_box(base + j * PA * (a_plane / 2) + q * (a_plane / 2), &p.tm_a, p.box_c0[ci], p.box_w0[ci],
                                             row0 * p.box_rs + p.box_r[ci], p.box_rs, q, &full_bar[stage]);
                        }
#pragma unroll
                        for (int q = 0; q < PB; ++q) tma_load_box(wbase + q * w_plane, &p.tm_b, nt * N, 0, row0, 1, q, &full_bar[stage]);
                    } else if (p.a_box) {                   // one box per plane: {64 B or 128 B of channels, pixels, grid rows}
#pragma unroll
                        for (int q = 0; q < PA; ++q)
                            tma_load_box(base + q * a_plane, &p.tm_a, p.box_c0[kc], p.box_w0[kc],
                                         (int)(mt * p.box_h) * p.box_rs + p.box_r[kc], p.box_rs, q, &full_bar[stage]);
                    } else if (p.a_tma) {
                        if (!WGRAD) {
                            tma_load_3d(base, &p.tm_a, kc * KC, (int)(mt * TILE_M), 0, &full_bar[stage]);        // A[row, k]
                        } else {                                    // A[site, kcol]: two blocks of 64 columns
                            tma_load_3d(base, &p.tm_a, (int)(mt * TILE_M), (int)site0, 0, &full_bar[stage]);
                            tma_load_3d(base + PA * (a_plane / 2), &p.tm_a, (int)(mt * TILE_M) + 64, (int)site0, 0, &full_bar[stage]);
                        }
                    }
                }
                if (!halo) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int pt = ptb + PROD_THREADS * h;
                        if (!WGRAD) xb_stage_fwd(g, s_units, pt, sites, kc, emit_a, emit_w);
                        else xb_stage_wgrad(g, s_units, pt, mt, site0, site_end, p.M, p.w_ld, nt * N, emit_a, emit_w);
                    }
                    // asynchronous publication: the barrier receives this thread's arrival when the copies issued above have
                    // landed - the producer never waits for its own loads, so up to `stages` chunks of loads are in flight
                    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(&full_bar[stage])) : "memory");
                }
                ++it;
            }
          }
        }
    } else {
        // ------------------------------------------------------------------ consumers: wgmma issue + epilogue
        //  A: halo     128-byte swizzle K-major window of the resident tile, K step 32 B, planes halo_plane apart
        //     cp.async no-swizzle canonical layout (conv_index.h), K step = two core matrices = 256 B
        //     TMA      128-byte swizzle.  K-major: rows of 128 B, K step 32 B.  MN-major (weight gradient): two blocks of 64
        //              columns, each [planes][64 sites][128 B]: plane stride a_plane/2, block stride PA*a_plane/2, K step 2048 B
        //  B: the first (PB - pa) planes, adjacent in the stage, are ONE operand of (PB - pa) * N rows (same three layouts;
        //     MN-major: one 64-column block per plane, blocks w_plane apart)
        // A descriptor = per-launch template (layout, LBO, SBO) + start address in 16-byte units; warpgroup wg reads rows
        // 64 wg .. 64 wg + 63 of the tile: 8192 bytes further in every layout but the MN-major TMA tile (the next 64-column block)
        const int wg = warp >> 2;
        uint64_t a_tmpl, b_tmpl;
        uint32_t a_ks, a_pl, b_ks, a_wg;                     // steps in 16-byte units: per K step of 16, per A plane; bytes per warpgroup
        if (halo) a_tmpl = make_desc_sw128(0, 16, 1024), a_ks = 32 >> 4, a_pl = halo_plane >> 4;
        else if (!p.a_tma) a_tmpl = make_desc(0, KC), a_ks = 256 >> 4, a_pl = a_plane >> 4;
        else if (!WGRAD) a_tmpl = make_desc_sw128(0, 16, 1024), a_ks = 32 >> 4, a_pl = a_plane >> 4;
        else a_tmpl = make_desc_sw128(0, PA * (a_plane / 2), 1024), a_ks = 2048 >> 4, a_pl = (a_plane / 2) >> 4;
        a_wg = (WGRAD && p.a_tma) ? (uint32_t)wg * PA * (a_plane / 2) : (uint32_t)wg * 8192u;
        if (!p.b_tma) b_tmpl = make_desc(0, KC), b_ks = 256 >> 4;
        else if (!WGRAD) b_tmpl = make_desc_sw128(0, 16, 1024), b_ks = 32 >> 4;
        else b_tmpl = make_desc_sw128(0, w_plane, 1024), b_ks = 2048 >> 4;
        // this thread's two rows of the tile and the first column of each 8-column block of its fragments
        const int rbase = 64 * wg + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
        float acc[PB * NC][16];
        uint32_t it = 0, tile_it = 0;
        for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x) {
          uint32_t halo_base = 0;
          int halo_s0 = 0;
          if (halo) {
              const uint32_t buf = tile_it & 1u;
              timed_wait(&a_full[buf], (tile_it >> 1) & 1u, 2);
              halo_base = smem_base + buf * a_buf_bytes;
              halo_s0 = (int)(w * TILE_M) - halo_row_lo(w) * p.halo_w;        // tile row of the site of MMA row 0
          }
          for (int sub = 0; sub < n_inner; ++sub) {
            const int n_chunks = chunks_of(w);
            const int64_t sp = WGRAD ? w / mn_tiles : 0;
            const int64_t rem = WGRAD ? w - sp * mn_tiles : w;
            const int64_t mt = halo ? w : rem / p.n_tiles;
            const int nt = halo ? sub : (int)(rem - mt * p.n_tiles);
            const int ncol = (halo && p.halo_same_cols) ? 0 : nt;             // column block of the output this item writes
            if (!WGRAD) {
                // the bias slice of this n tile (only the consumer warps read / write s_bias; named barrier 1)
                asm volatile("bar.sync 1, %0;" ::"n"(CONS_WARPS * 32) : "memory");
                for (int i = tid; i < N; i += CONS_WARPS * 32) s_bias[i] = p.bias ? p.bias[ncol * N + i] : 0.f;
            }
            uint32_t scale_d = 0;
            int prev_stage = -1;
            for (int kc = 0; kc < n_chunks; ++kc) {
                const int stage = (int)(it % (uint32_t)S);
                timed_wait(&full_bar[stage], (it / (uint32_t)S) & 1u, 0);
                fence_proxy_async();       // the stage was written by cp.async (generic proxy); the MMA reads it through the async proxy
                const uint32_t base = smem_base + ring_off + (uint32_t)stage * stage_bytes;
                const uint32_t w_addr = base + (halo ? 0u : PA * a_plane);
                const uint32_t a_addr = a_wg + (halo ? halo_base + (uint32_t)(halo_s0 + p.halo_shift[sub * p.halo_chunks + kc]) * 128u : base);
                // start addresses stay below 2^18 bytes: adding 16-byte units to the template never carries out of the field
                const uint64_t a0 = a_tmpl + (uint64_t)(a_addr >> 4), b0 = b_tmpl + (uint64_t)(w_addr >> 4);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < KC / 16; ++ks) {
                    // A plane pa x B planes 0 .. PB-1-pa -> accumulator groups pa .. PB-1.
                    // pa = 0 covers every group, so its first instruction of a work item (scale_d = 0) initialises them all.
                    const uint64_t da = a0 + (uint64_t)(ks * a_ks), db = b0 + (uint64_t)(ks * b_ks);
                    mma_plane<TR, PB, NC, 0>(acc, da, db, scale_d);
                    if (PA > 1) mma_plane<TR, PB, NC, (PA > 1 ? 1 : 0)>(acc, da + a_pl, db, 1u);
                    if (PA > 2) mma_plane<TR, PB, NC, (PA > 2 ? 2 : 0)>(acc, da + 2 * a_pl, db, 1u);
                    scale_d = 1;
                }
                wgmma_commit();
                // the group before this one has retired: its stage is free
                wgmma_wait<1>();
                if (prev_stage >= 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
                }
                prev_stage = stage;
                ++it;
            }
            wgmma_wait<0>();
            if (prev_stage >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
            }
            if (!WGRAD) asm volatile("bar.sync 1, %0;" ::"n"(CONS_WARPS * 32) : "memory");     // s_bias written
            // ---- epilogue on the fragments: rows rbase (h = 0) and rbase + 8 (h = 1)
            bool live[2];
            int64_t orow[2] = {0, 0}, mrow[2] = {0, 0};                       // element offsets of the output row / of its mask row
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                if (halo) {
                    const int64_t P = mt * TILE_M + r;                         // position in the haloed raster
                    const uint32_t R = xb_div((uint32_t)P, p.halo_div_w);      // merged (image, padded row) index
                    const int x = (int)((uint32_t)P - R * (uint32_t)p.halo_w) + p.halo_w0;
                    const int b = (int)xb_div(R, p.box_div_hp), y = (int)(R - (uint32_t)b * (uint32_t)p.box_hp);
                    live[h] = P < p.halo_positions && x >= 0 && x <= p.sub_x1[nt] && y >= p.box_y0 && y <= p.sub_y1[nt];
                    if (live[h]) {
                        const int64_t orw = (int64_t)b * p.out_H + ((y - p.box_y0) * p.oys + p.sub_oy0[nt]);
                        const int ox = x * p.oxs + p.sub_ox0[nt];
                        orow[h] = (orw * p.out_W + ox) * p.out_ld + p.out_c0 + (int64_t)ncol * N;
                        mrow[h] = (orw * p.mask_W + ox + p.mask_x0) * p.mask_ld + p.mask_c0 + (int64_t)ncol * N;
                    }
                } else if (!WGRAD && p.a_box) {
                    const int gr = (int)xb_div((uint32_t)r, p.box_div_w), x = r - gr * p.box_w;
                    const int64_t R = mt * p.box_h + gr;                       // merged (image, padded row) index
                    const int b = (int)xb_div((uint32_t)R, p.box_div_hp), y = (int)(R - (int64_t)b * p.box_hp);
                    live[h] = r < box_rows && b < g.B && y >= p.box_y0 && y <= p.box_y1;
                    if (live[h]) {
                        const int64_t orw = (int64_t)b * p.out_H + ((y - p.box_y0) * p.oys + p.oy0);
                        const int ox = x * p.oxs + p.ox0;
                        orow[h] = (orw * p.out_W + ox) * p.out_ld + p.out_c0 + (int64_t)nt * N;
                        mrow[h] = (orw * p.mask_W + ox + p.mask_x0) * p.mask_ld + p.mask_c0 + (int64_t)nt * N;
                    }
                } else if (!WGRAD) {
                    const int64_t m = mt * TILE_M + r;
                    live[h] = m < p.M;
                    if (live[h]) {
                        int b, y, x;
                        xb_conv_site(g, m, b, y, x);
                        const int64_t opix = ((int64_t)b * p.out_H + (y * p.oys + p.oy0)) * p.out_W + (x * p.oxs + p.ox0);
                        orow[h] = opix * p.out_ld + p.out_c0 + (int64_t)nt * N;
                        mrow[h] = opix * p.mask_ld + p.mask_c0 + (int64_t)nt * N;
                    }
                } else {
                    const int64_t kcol = mt * TILE_M + r;
                    live[h] = kcol < K;
                    orow[h] = ((sp * K + kcol) * p.n_tiles + nt) * (int64_t)N;       // partials [splits, K, N_total]
                }
            }
#pragma unroll
            for (int cc = 0; cc < NC; ++cc) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int c = 32 * cc + 8 * i + cq;                        // columns c, c + 1
                    float cs[2] = {0.f, 0.f};
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float v[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            v[e] = acc[(PB - 1) * NC + cc][4 * i + 2 * h + e];     // smallest group first
#pragma unroll
                            for (int gq = PB - 2; gq >= 0; --gq) v[e] += acc[gq * NC + cc][4 * i + 2 * h + e];
                            if (!WGRAD) {
                                v[e] += s_bias[c + e];
                                if (p.relu) v[e] = fmaxf(v[e], 0.f);
                            }
                        }
                        if (!WGRAD && p.mask && live[h]) {
                            // bf16 > 0  <=>  sign bit clear and not (+)zero
                            const uint32_t mw = *reinterpret_cast<const uint32_t *>(p.mask + mrow[h] + c);
                            const uint32_t lo16 = mw & 0xffffu, hi16 = mw >> 16;
                            if (!(lo16 != 0u && lo16 < 0x8000u)) v[0] = 0.f;
                            if (!(hi16 != 0u && hi16 < 0x8000u)) v[1] = 0.f;
                        }
                        if (live[h]) {
                            if (p.out_f32) *reinterpret_cast<float2 *>(p.out_f32 + orow[h] + c) = make_float2(v[0], v[1]);
                            if (!WGRAD && p.p_out > 0) {
                                __nv_bfloat16 q0[3], q1[3];
                                split3_bf16(v[0], q0[0], q0[1], q0[2]);
                                split3_bf16(v[1], q1[0], q1[1], q1[2]);
#pragma unroll
                                for (int q = 0; q < 3; ++q)
                                    if (q < p.p_out) *reinterpret_cast<uint32_t *>(p.out[q] + orow[h] + c) = pack2(q0[q], q1[q]);
                            }
                            cs[0] += v[0], cs[1] += v[1];
                        }
                    }
                    if (!WGRAD && p.colsum) {
                        // column sums over the warp's 16 rows: the 8 lanes that share (lane & 3) hold the same columns
#pragma unroll
                        for (int off = 4; off <= 16; off <<= 1) {
                            cs[0] += __shfl_xor_sync(0xffffffffu, cs[0], off);
                            cs[1] += __shfl_xor_sync(0xffffffffu, cs[1], off);
                        }
                        if (lane < 4) s_colsum[warp][c] = cs[0], s_colsum[warp][c + 1] = cs[1];
                    }
                }
            }
            if (!WGRAD && p.colsum) {
                asm volatile("bar.sync 1, %0;" ::"n"(CONS_WARPS * 32) : "memory");
                for (int i = tid; i < N; i += CONS_WARPS * 32) {          // fixed order: deterministic
                    float s = s_colsum[0][i];
#pragma unroll
                    for (int q = 1; q < CONS_WARPS; ++q) s += s_colsum[q][i];
                    p.colsum[(mt * p.n_tiles + nt) * (int64_t)N + i] = s;
                }
            }
          }
          if (halo) {
              __syncwarp();                                   // every MMA of this tile has retired (wait above)
              if (lane == 0) mbar_arrive(&a_empty[tile_it & 1u]);
              ++tile_it;
          }
        }
    }
    if (p.timing && blockIdx.x < 160) {
        const unsigned long long tot = clock64() - t_begin;
        unsigned long long *o = xb_k12_timing[blockIdx.x];
        if (tid == 0) o[0] = tot, o[1] = t_wait[0], o[3] = t_wait[2];
        if (warp == CONS_WARPS && lane == 0) o[4] = tot, o[5] = t_wait[0], o[6] = t_wait[1];
    }
}

// weight-gradient finish: sum the split partials [splits, K, N] in a fixed order and scatter to torch's [N, C, KH, KW]
// (column k = (kh, kw, c) of the packed layout -> xb_pack_weight_src); accumulate != 0 adds to dw (autograd .grad).
// A block owns E = 256 / lanes consecutive (k, n) elements - coalesced rows of the partial matrices - and `lanes` threads
// per element walk the splits interleaved.  Many splits (bias-gradient partials: one row per M tile) are first folded in
// place, group g of `group` consecutive splits into its first row (blockIdx.y = g), then the group rows are summed.
__device__ __forceinline__ float reduce_splits(const float *__restrict__ ws, int64_t total, int64_t j, int first, int last, int step,
                                               int lanes, int E, float *part) {
    const int e = threadIdx.x % E, l = threadIdx.x / E;
    float s = 0.f;
    if (j < total)
        for (int sp = first + l * step; sp < last; sp += lanes * step) s += ws[(int64_t)sp * total + j];
    part[threadIdx.x] = s;
    __syncthreads();
    if (l == 0)
        for (int q = 1; q < lanes; ++q) s += part[e + q * E];
    return s;
}

__global__ void __launch_bounds__(256) wgrad_fold_kernel(float *__restrict__ ws, int splits, int group, int lanes, int64_t total) {
    __shared__ float part[256];
    const int E = 256 / lanes;
    const int64_t j = (int64_t)blockIdx.x * E + threadIdx.x % E;
    const int first = blockIdx.y * group, last = min(first + group, splits);
    const float s = reduce_splits(ws, total, j, first, last, 1, lanes, E, part);
    if (threadIdx.x < E && j < total) ws[(int64_t)first * total + j] = s;     // read only by this thread before
}

// the reduction for weights with many taps (see xb_pack_tiled): tile = 32 n x 2 c x HW; partial rows [k][n0 .. n0+31] are read
// coalesced, torch's dw[n][c][hw] is written in runs of HW
__global__ void __launch_bounds__(256) wgrad_reduce_tiled_kernel(const float *__restrict__ ws, int splits, int step, int N, int C, int HW,
                                                                 float scale, float *__restrict__ dw, int accumulate) {
    __shared__ float tile[2 * 128 * 33];
    const int cpairs = C / 2, n0 = (int)(blockIdx.x / cpairs) * 32, c0 = (int)(blockIdx.x % cpairs) * 2, run = 2 * HW;
    const int64_t total = (int64_t)N * C * HW;
    for (int i = threadIdx.x; i < 32 * run; i += 256) {
        const int r = i >> 5, nl = i & 31, cl = r / HW, hw = r - cl * HW;
        const int64_t j = ((int64_t)hw * C + c0 + cl) * N + n0 + nl;
        float s = 0.f;
        for (int sp = 0; sp < splits; sp += step) s += ws[(int64_t)sp * total + j];
        tile[r * 33 + nl] = __fmul_rn(s, scale);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * run; i += 256) {
        const int nl = i / run, r = i - nl * run;
        const int64_t dst = ((int64_t)(n0 + nl) * C + c0) * HW + r;
        const float v = tile[r * 33 + nl];
        dw[dst] = accumulate ? dw[dst] + v : v;
    }
}

__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float *__restrict__ ws, int splits, int step, int lanes, int N, int C,
                                                           int KH, int KW, float scale, float *__restrict__ dw, int accumulate) {
    __shared__ float part[256];
    const int64_t K = (int64_t)C * KH * KW, total = (int64_t)N * K;
    const int E = 256 / lanes;
    const int64_t j = (int64_t)blockIdx.x * E + threadIdx.x % E;
    float s = reduce_splits(ws, total, j, 0, splits, step, lanes, E, part);
    if (threadIdx.x < E && j < total) {
        s = __fmul_rn(s, scale);
        const int64_t k = j / N, n = j - k * N;
        const int64_t dst = xb_pack_weight_src(n * K + k, C, KH, KW);     // packed index [N, (kh, kw, c)] -> [N, C, KH, KW]
        dw[dst] = accumulate ? dw[dst] + s : s;
    }
}

// ---------------------------------------------------------------- operand preparation (HBM-bound, elementwise)
// planes: out is [P, n] bf16; plane 0 = bf16(x), plane q = bf16 of the residual left by planes < q
template <int P>
__global__ void __launch_bounds__(256) split_bf16_kernel(const float *__restrict__ x, int64_t n8, int64_t n,
                                                         __nv_bfloat16 *__restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
        float v[8];
        const int64_t e = i * 8;
        const bool full = e + 8 <= n;
        if (full) {
            const float4 a = reinterpret_cast<const float4 *>(x + e)[0], b = reinterpret_cast<const float4 *>(x + e)[1];
            v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = b.x, v[5] = b.y, v[6] = b.z, v[7] = b.w;
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = e + j < n ? x[e + j] : 0.f;
        }
#pragma unroll
        for (int q = 0; q < P; ++q) {
            __nv_bfloat16 h[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                h[j] = __float2bfloat16_rn(v[j]);
                v[j] -= __bfloat162float(h[j]);
            }
            __nv_bfloat16 *dst = out + (int64_t)q * n + e;
            if (full && ((n & 7) == 0)) {
                *reinterpret_cast<uint4 *>(dst) = make_uint4(pack2(h[0], h[1]), pack2(h[2], h[3]), pack2(h[4], h[5]), pack2(h[6], h[7]));
            } else {
                for (int j = 0; j < 8 && e + j < n; ++j) dst[j] = h[j];
            }
        }
    }
}

// torch weight [N, C, KH, KW] (also a Linear over a flattened [C, H, W] feature map) -> [P, N, (kh, kw, c)] bf16 planes
template <int P>
__global__ void __launch_bounds__(256) pack_weight_kernel(const float *__restrict__ w, int N, int C, int KH, int KW,
                                                          float scale, __nv_bfloat16 *__restrict__ out) {
    const int64_t total = (int64_t)N * C * KH * KW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        float v = __fmul_rn(w[xb_pack_weight_src(i, C, KH, KW)], scale);   // scale 1/255: the layer reads raw uint8 pixels
#pragma unroll
        for (int q = 0; q < P; ++q) {
            const __nv_bfloat16 h = __float2bfloat16_rn(v);
            out[(int64_t)q * total + i] = h;
            v -= __bfloat162float(h);
        }
    }
}

// every operand form of several weights in ONE launch (the per-update operand preparation of an encoder: forward packs,
// transposed packs and data-gradient matrices); a block works on one job, jobs own consecutive block ranges
struct PackJobs {
    XbPackJob job[XB_PACK_MAX_JOBS];
    unsigned first_block[XB_PACK_MAX_JOBS + 1];
    int tiled[XB_PACK_MAX_JOBS];           // weights with many taps (a Linear over a [C, H, W] map): transpose through shared memory
    int n;
};
// [N, C, HW] <-> [N, (hw, c)] is a C x HW transpose per n with strides of HW elements: element-wise it touches one 32-byte
// sector per 4-byte value on one side (the 512 x 6400 Linear layer is the case that matters).  Tiles through shared
// memory make both sides coalesced: mode 0 one n (C*HW values) per block; mode 1 / the weight-gradient reduction a tile of
// 32 n x 2 c x HW values (rows of 32 n on the (hw, c)-major side, runs of HW on torch's side).
constexpr int PACK_TILE_MAX = 8192;        // floats of shared memory per block
__host__ __device__ inline bool xb_pack_tiled(int mode, int N, int C, int HW) {
    if (HW < 32) return false;
    if (mode == 0) return C * HW <= PACK_TILE_MAX - C;
    if (mode == 1 || mode == 3) return N % 32 == 0 && C % 2 == 0 && 2 * HW * 33 <= PACK_TILE_MAX;
    return false;
}

__global__ void __launch_bounds__(256) pack_jobs_kernel(const __grid_constant__ PackJobs pj) {
    int ji = 0;
    while (ji + 1 < pj.n && blockIdx.x >= pj.first_block[ji + 1]) ++ji;
    const XbPackJob &J = pj.job[ji];
    const int64_t K = (int64_t)J.C * J.KH * J.KW, total = J.mode == 2 ? (int64_t)J.C * J.n_taps * J.N : (int64_t)J.N * K;
    __shared__ float tile[PACK_TILE_MAX];
    if (pj.tiled[ji]) {
        const int HW = J.KH * J.KW, C = J.C;
        const unsigned tb = blockIdx.x - pj.first_block[ji];
        __nv_bfloat16 *out = (__nv_bfloat16 *)J.out;
        if (J.mode == 0) {
            // one n: torch's [C][HW] run is read in order, written as [(hw, c)]; shared row pitch HW + 1
            const int64_t n = tb;
            const float *src = J.w + n * K;
            for (int i = threadIdx.x; i < (int)K; i += 256) tile[(i / HW) * (HW + 1) + i % HW] = src[i];
            __syncthreads();
            for (int i = threadIdx.x; i < (int)K; i += 256) {
                const int hw = i / C, c = i - hw * C;
                float v = __fmul_rn(tile[c * (HW + 1) + hw], J.scale);
                for (int q = 0; q < J.planes; ++q) {
                    const __nv_bfloat16 h = __float2bfloat16_rn(v);
                    out[(int64_t)q * total + n * K + i] = h;
                    v -= __bfloat162float(h);
                }
            }
        } else {
            // 32 n x 2 c x HW: read runs of 2*HW of torch's layout per n, write rows of 32 n at k = hw*C + c
            const int cpairs = C / 2, n0 = (int)(tb / cpairs) * 32, c0 = (int)(tb % cpairs) * 2, run = 2 * HW;
            for (int i = threadIdx.x; i < 32 * run; i += 256) {
                const int nl = i / run, r = i - nl * run;
                tile[r * 33 + nl] = J.w[((int64_t)(n0 + nl) * C + c0) * HW + r];
            }
            __syncthreads();
            for (int i = threadIdx.x; i < 32 * run; i += 256) {
                const int r = i >> 5, nl = i & 31, cl = r / HW, hw = r - cl * HW;
                float v = __fmul_rn(tile[r * 33 + nl], J.scale);
                const int64_t o = ((int64_t)hw * C + c0 + cl) * J.N + n0 + nl;
                for (int q = 0; q < J.planes; ++q) {
                    const __nv_bfloat16 h = __float2bfloat16_rn(v);
                    out[(int64_t)q * total + o] = h;
                    v -= __bfloat162float(h);
                }
            }
        }
        return;
    }
    const int64_t i = (int64_t)(blockIdx.x - pj.first_block[ji]) * 256 + threadIdx.x;
    if (i >= total) return;
    int64_t src;
    if (J.mode == 0) {
        src = xb_pack_weight_src(i, J.C, J.KH, J.KW);                       // [N][(kh, kw, c)]
    } else if (J.mode == 1) {
        const int64_t k = i / J.N, n = i - k * J.N;                        // [(kh, kw, c)][N]
        src = xb_pack_weight_src(n * K + k, J.C, J.KH, J.KW);
    } else {
        const int64_t tn = (int64_t)J.n_taps * J.N, c = i / tn, r = i - c * tn;   // [C][(tap, n)]
        const int t = (int)(r / J.N), n = (int)(r - (int64_t)t * J.N);
        src = (((int64_t)n * J.C + c) * J.KH + J.kh[t]) * J.KW + J.kw[t];
    }
    float v = __fmul_rn(J.w[src], J.scale);
    __nv_bfloat16 *out = (__nv_bfloat16 *)J.out;
    for (int q = 0; q < J.planes; ++q) {
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        out[(int64_t)q * total + i] = h;
        v -= __bfloat162float(h);
    }
}

// ---------------------------------------------------------------- TMA descriptors (host)
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)ptr;
        cudaGetLastError();
    }
    return fn;
}
// XB_K12_TMA=0 keeps every operand on the cp.async path (the one the host emulator models)
bool tma_enabled() {
    static int on = -1;
    if (on < 0) {
        const char *e = getenv("XB_K12_TMA");
        on = (e && e[0] == '0') ? 0 : 1;
    }
    return on == 1;
}
// bf16 tensor [planes][rows][cols] (cols contiguous, row_stride / plane_stride in elements), tiles {64 cols, box_rows, planes},
// 128-byte swizzle, zero fill outside [rows, cols]
bool make_tmap(CUtensorMap *tm, const void *base, int64_t cols, int64_t rows, int planes, int64_t row_stride,
               int64_t plane_stride, int box_rows) {
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) return false;
    if (((uintptr_t)base & 15) || (row_stride * 2) % 16 || (plane_stride * 2) % 16 || box_rows > 256) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)planes};
    const cuuint64_t strides[2] = {(cuuint64_t)row_stride * 2, (cuuint64_t)(planes > 1 ? plane_stride : row_stride * rows) * 2};
    const cuuint32_t box[3] = {64, (cuuint32_t)box_rows, (cuuint32_t)planes};
    const cuuint32_t estr[3] = {1, 1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(base), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// bf16 activation tensor [planes][rows][pixels][channels] (padded-row layout, rows = images x padded rows per image merged),
// boxes of {64 channels, box_px pixels, box_h rows of ONE row phase, one plane}, 128-byte swizzle
bool make_tmap_box(CUtensorMap *tm, const void *base, int C, int W, int64_t rows, int planes, int64_t plane_stride, int box_c,
                   int box_px, int box_h, int row_step) {
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) return false;
    if (((uintptr_t)base & 15) || (C * 2) % 16 || (plane_stride * 2) % 16 || rows % row_step != 0) return false;
    if (box_c * 2 != 128 || box_px > 256 || box_h > 256) return false;     // 128-byte inner box: one shared-memory row per pixel
    const cuuint64_t S = (cuuint64_t)row_step;
    // {channels, pixels, row phase, row / S, plane}
    const cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, S, (cuuint64_t)rows / S, (cuuint64_t)planes};
    const cuuint64_t row_b = (cuuint64_t)W * C * 2;
    const cuuint64_t strides[4] = {(cuuint64_t)C * 2, row_b, S * row_b, (cuuint64_t)(planes > 1 ? plane_stride : rows * W * C) * 2};
    const cuuint32_t box[5] = {(cuuint32_t)box_c, (cuuint32_t)box_px, 1, (cuuint32_t)box_h, 1};
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void *>(base), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

int fill_params(ConvParams &p, int pa, int pb, const void *in, int64_t in_plane, const void *w, int64_t w_plane, int B,
                int IH, int IW, int C, int OY, int OX, int sy, int sx, int T, const int8_t *dy, const int8_t *dx, int N,
                int n_tile) {
    if (pa < 1 || pb > 3 || pa > pb) return XB_EINVAL;
    if (!in || !w || !dy || !dx) return XB_EINVAL;
    if (B <= 0 || IH <= 0 || IW <= 0 || OY <= 0 || OX <= 0 || sy <= 0 || sx <= 0 || T <= 0 || N <= 0 || n_tile <= 0)
        return XB_EINVAL;
    // the register accumulators of one consumer thread: pb * n_tile / 2 floats (pb * n_tile <= 256, n_tile a multiple of 32)
    if (T > XB_CONV_MAX_TAPS || n_tile % 32 != 0 || N % n_tile != 0 || pb * n_tile > 256 || C % 8 != 0) return XB_ERANGE;
    if ((int64_t)T * C > 8 * XB_CONV_MAX_UNITS || (int64_t)B * OY * OX >= (int64_t)1 << 31) return XB_ERANGE;   // tap table, 32-bit sites
    if (!xb_aligned(in, 16) || !xb_aligned(w, 16) || in_plane % 8 != 0 || w_plane % 8 != 0) return XB_EALIGN;
    p.g.B = B, p.g.IH = IH, p.g.IW = IW, p.g.C = C, p.g.OY = OY, p.g.OX = OX, p.g.sy = sy, p.g.sx = sx, p.g.T = T, p.g.N = n_tile;
    for (int t = 0; t < XB_CONV_MAX_TAPS; ++t) p.g.dy[t] = t < T ? dy[t] : 0, p.g.dx[t] = t < T ? dx[t] : 0;
    xb_geom_finish(p.g);
    const __nv_bfloat16 *ib = (const __nv_bfloat16 *)in, *wb = (const __nv_bfloat16 *)w;
    for (int q = 0; q < 3; ++q) p.in[q] = q < pa ? ib + q * in_plane : nullptr, p.w[q] = q < pb ? wb + q * w_plane : nullptr;
    p.M = (int64_t)B * OY * OX;
    p.n_tiles = N / n_tile;
    const uint32_t stage_bytes = pa * xb_conv_a_plane_bytes() + pb * xb_conv_w_plane_bytes(n_tile);
    int stages = (int)((200u * 1024u) / stage_bytes);
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    if (stages < 2) return XB_ERANGE;
    p.stages = stages;
    p.a_tma = p.b_tma = p.a_box = p.a_halo = 0;
    p.dyn_smem = 0;
    {
        static int timing = -1;
        if (timing < 0) {
            const char *e = getenv("XB_K12_TIMING");
            timing = (e && atoi(e) != 0) ? 1 : 0;
        }
        p.timing = timing;
    }
    p.box_w = p.box_h = p.box_hp = 1, p.box_y0 = p.box_y1 = 0, p.box_rs = 1, p.box_chunks = 0;
    return XB_OK;
}

template <bool WGRAD, int PA, int PB, int NC>
int launch_pp(const ConvParams &p, int64_t work, void *stream) {
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(conv_tc_kernel<WGRAD, PA, PB, NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, XB_K12_MAX_DYN_SMEM);
        attr = true;
    }
    const int grid = (int)(work < xb_sm_count() ? work : xb_sm_count());
    const size_t smem = p.dyn_smem ? p.dyn_smem : (size_t)p.stages * (PA * xb_conv_a_plane_bytes() + PB * xb_conv_w_plane_bytes(p.g.N));
    conv_tc_kernel<WGRAD, PA, PB, NC><<<grid, THREADS, smem, (cudaStream_t)stream>>>(p);
    return xb_launch_status();
}

// the tile width N = 32 NC is a template parameter: the accumulators are registers (PB * NC blocks of 32 columns, at most 8)
template <bool WGRAD, int PA, int PB, int NC = 1>
int launch_n(const ConvParams &p, int64_t work, void *stream) {
    if constexpr (PB * NC > 8) {
        return XB_ERANGE;
    } else {
        if (p.g.N == 32 * NC) return launch_pp<WGRAD, PA, PB, NC>(p, work, stream);
        return launch_n<WGRAD, PA, PB, NC + 1>(p, work, stream);
    }
}

template <bool WGRAD>
int launch(int pa, int pb, const ConvParams &p, int64_t work, void *stream) {
    if (pa == 1 && pb == 1) return launch_n<WGRAD, 1, 1>(p, work, stream);
    if (pa == 1 && pb == 2) return launch_n<WGRAD, 1, 2>(p, work, stream);
    if (pa == 1 && pb == 3) return launch_n<WGRAD, 1, 3>(p, work, stream);
    if (pa == 2 && pb == 2) return launch_n<WGRAD, 2, 2>(p, work, stream);
    if (pa == 2 && pb == 3) return launch_n<WGRAD, 2, 3>(p, work, stream);
    if (pa == 3 && pb == 3) return launch_n<WGRAD, 3, 3>(p, work, stream);
    return XB_EINVAL;
}

}  // namespace

extern "C" int xb_split_bf16(const float *x, int64_t n, int planes, void *out, void *stream) {
    if (!x || !out || n <= 0 || planes < 1 || planes > 3) return XB_EINVAL;
    if (!xb_aligned(x, 16) || !xb_aligned(out, 16)) return XB_EALIGN;
    const int64_t n8 = (n + 7) / 8;
    int64_t want = (n8 + 255) / 256;
    const int grid = (int)(want < (int64_t)xb_sm_count() * 8 ? want : (int64_t)xb_sm_count() * 8);
    if (planes == 1) split_bf16_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(x, n8, n, (__nv_bfloat16 *)out);
    else if (planes == 2) split_bf16_kernel<2><<<grid, 256, 0, (cudaStream_t)stream>>>(x, n8, n, (__nv_bfloat16 *)out);
    else split_bf16_kernel<3><<<grid, 256, 0, (cudaStream_t)stream>>>(x, n8, n, (__nv_bfloat16 *)out);
    return xb_launch_status();
}

extern "C" int xb_pack_conv_weight(const float *w, int N, int C, int KH, int KW, int planes, float scale, void *out,
                                   void *stream) {
    if (!w || !out || N <= 0 || C <= 0 || KH <= 0 || KW <= 0 || planes < 1 || planes > 3) return XB_EINVAL;
    const int64_t total = (int64_t)N * C * KH * KW;
    int64_t want = (total + 255) / 256;
    const int grid = (int)(want < (int64_t)xb_sm_count() * 8 ? want : (int64_t)xb_sm_count() * 8);
    cudaStream_t s = (cudaStream_t)stream;
    if (planes == 1) pack_weight_kernel<1><<<grid, 256, 0, s>>>(w, N, C, KH, KW, scale, (__nv_bfloat16 *)out);
    else if (planes == 2) pack_weight_kernel<2><<<grid, 256, 0, s>>>(w, N, C, KH, KW, scale, (__nv_bfloat16 *)out);
    else pack_weight_kernel<3><<<grid, 256, 0, s>>>(w, N, C, KH, KW, scale, (__nv_bfloat16 *)out);
    return xb_launch_status();
}

extern "C" int xb_pack_weights(const XbPackJob *jobs, int n_jobs, void *stream) {
    if (!jobs || n_jobs <= 0 || n_jobs > XB_PACK_MAX_JOBS) return XB_EINVAL;
    PackJobs pj;
    pj.n = n_jobs;
    uint64_t blocks = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const XbPackJob &J = jobs[j];
        if (!J.w || !J.out || J.N <= 0 || J.C <= 0 || J.KH <= 0 || J.KW <= 0 || J.planes < 1 || J.planes > 3 || J.mode < 0 ||
            J.mode > 2)
            return XB_EINVAL;
        if (J.mode == 2) {
            if (J.n_taps <= 0 || J.n_taps > XB_PACK_MAX_TAPS) return XB_ERANGE;
            for (int t = 0; t < J.n_taps; ++t)
                if (J.kh[t] < 0 || J.kh[t] >= J.KH || J.kw[t] < 0 || J.kw[t] >= J.KW) return XB_ERANGE;
        }
        if (!xb_aligned(J.out, 2) || !xb_aligned(J.w, 4)) return XB_EALIGN;
        const int64_t total = J.mode == 2 ? (int64_t)J.C * J.n_taps * J.N : (int64_t)J.N * J.C * J.KH * J.KW;
        pj.job[j] = J;
        pj.first_block[j] = (unsigned)blocks;
        pj.tiled[j] = (J.mode != 2 && xb_pack_tiled(J.mode, J.N, J.C, J.KH * J.KW)) ? 1 : 0;
        if (pj.tiled[j]) blocks += J.mode == 0 ? (uint64_t)J.N : (uint64_t)(J.N / 32) * (uint64_t)(J.C / 2);
        else
        blocks += (uint64_t)((total + 255) / 256);
        if (blocks > 0x7fffffffull) return XB_ERANGE;
    }
    pj.first_block[n_jobs] = (unsigned)blocks;
    pack_jobs_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(pj);
    return xb_launch_status();
}

extern "C" int xb_gemm_gather_tc(int planes_a, int planes_b, const void *in, int64_t in_plane, const void *w, int64_t w_plane,
                                 const float *bias, const void *relu_mask, int64_t mask_ld, int mask_c0, int B, int IH, int IW,
                                 int C, int OY, int OX, int sy, int sx, int T, const int8_t *dy, const int8_t *dx, int N,
                                 int n_tile, int relu, void *out_planes, int64_t out_plane, int planes_out, float *out_f32,
                                 int out_H, int out_W, int oys, int oxs, int oy0, int ox0, int64_t out_ld, int out_c0,
                                 float *colsum, void *stream) {
    ConvParams p;
    const int rc = fill_params(p, planes_a, planes_b, in, in_plane, w, w_plane, B, IH, IW, C, OY, OX, sy, sx, T, dy, dx, N, n_tile);
    if (rc != XB_OK) return rc;
    if (!out_planes && !out_f32) return XB_EINVAL;
    if (out_planes && (planes_out < 1 || planes_out > 3)) return XB_EINVAL;
    if (((int64_t)T * C) % XB_CONV_KC != 0) return XB_ERANGE;
    if (out_H <= 0 || out_W <= 0 || oys <= 0 || oxs <= 0 || oy0 < 0 || ox0 < 0 || (OY - 1) * oys + oy0 >= out_H ||
        (OX - 1) * oxs + ox0 >= out_W || out_c0 < 0 || out_ld < (int64_t)out_c0 + N)
        return XB_EINVAL;
    if (out_ld % 8 != 0 || out_c0 % 8 != 0 || out_plane % 8 != 0) return XB_EALIGN;   // 16-byte row segments
    if ((out_planes && !xb_aligned(out_planes, 16)) || (out_f32 && !xb_aligned(out_f32, 16)) ||
        (relu_mask && !xb_aligned(relu_mask, 16)))
        return XB_EALIGN;
    if (mask_ld != 0 && (mask_ld % 8 != 0 || mask_c0 % 8 != 0 || mask_c0 < 0 || mask_ld < (int64_t)mask_c0 + N)) return XB_EALIGN;
    p.bias = bias;
    p.mask = (const __nv_bfloat16 *)relu_mask;
    p.mask_W = out_W, p.mask_x0 = 0;
    p.mask_ld = mask_ld != 0 ? mask_ld : out_ld, p.mask_c0 = mask_ld != 0 ? mask_c0 : out_c0;
    p.colsum = colsum;
    __nv_bfloat16 *ob = (__nv_bfloat16 *)out_planes;
    p.p_out = ob ? planes_out : 0;
    for (int q = 0; q < 3; ++q) p.out[q] = (ob && q < planes_out) ? ob + q * out_plane : nullptr;
    p.out_f32 = out_f32;
    p.relu = relu;
    p.out_H = out_H, p.out_W = out_W, p.oys = oys, p.oxs = oxs, p.oy0 = oy0, p.ox0 = ox0;
    p.out_ld = out_ld, p.out_c0 = out_c0;
    p.splits = 1, p.sites_per_split = 0, p.w_ld = 0;
    if (tma_enabled()) {
        const int64_t K = (int64_t)T * C;
        // weights [planes_b][N][K]: tiles of {64 k, n_tile rows, all planes}
        p.b_tma = make_tmap(&p.tm_b, w, K, N, planes_b, K, w_plane, n_tile) ? 1 : 0;
        // a Linear layer's input [planes_a][B][C] is a plain matrix too: tiles of {64 k, 128 rows, all planes}
        if (T == 1 && IH == 1 && IW == 1 && OY == 1 && OX == 1)
            p.a_tma = make_tmap(&p.tm_a, in, C, B, planes_a, C, in_plane, TILE_M) ? 1 : 0;
    }
    const int64_t tiles = (p.M + TILE_M - 1) / TILE_M * p.n_tiles;
    return launch<false>(planes_a, planes_b, p, tiles, stream);
}

// The same GEMM with the A operand of a convolution fetched by TMA boxes from a padded-row activation tensor (see ConvParams
// a_box); needs a driver that resolves cuTensorMapEncodeTiled (returns XB_EINVAL otherwise - there is no silent fallback).
extern "C" int xb_gemm_box_tc(int planes_a, int planes_b, const void *in, int64_t in_plane, int C, int W, int64_t in_rows,
                              int box_c, int box_px, int box_h, int row_step, int n_chunks, const int16_t *c0,
                              const int16_t *w0, const int16_t *r0, const void *w, int64_t w_plane, const float *bias,
                              const void *relu_mask, int mask_W, int mask_x0, int B, int hp, int y0, int y1, int N, int n_tile,
                              int relu,
                              void *out_planes, int64_t out_plane, int planes_out, float *out_f32, int out_H, int out_W,
                              int oys, int oxs, int oy0, int ox0, int64_t out_ld, int out_c0, float *colsum, void *stream) {
    if (!c0 || !w0 || !r0 || n_chunks <= 0 || n_chunks > 16) return XB_EINVAL;
    if (box_c != 64 || box_px <= 0 || box_h <= 0 || row_step <= 0 || row_step > 8) return XB_EINVAL;
    const int box_w = box_px;                               // sites (GEMM rows) per grid row: one 64-channel pixel each
    if (box_w * box_h > TILE_M || hp <= 0 || y0 < 0 || y1 < y0 || y1 >= hp || B <= 0) return XB_ERANGE;
    ConvParams p;
    // geometry fields that the generic checks read: one "tap" of 64 channels per chunk
    int8_t zero[XB_CONV_MAX_TAPS] = {0};
    const int rc = fill_params(p, planes_a, planes_b, in, in_plane, w, w_plane, B, 1, 1, 64, 1, 1, 1, 1, n_chunks, zero, zero, N,
                               n_tile);
    if (rc != XB_OK) return rc;
    if (!out_planes && !out_f32) return XB_EINVAL;
    if (out_planes && (planes_out < 1 || planes_out > 3)) return XB_EINVAL;
    if (out_ld % 8 != 0 || out_c0 % 8 != 0 || out_plane % 8 != 0) return XB_EALIGN;
    if ((out_planes && !xb_aligned(out_planes, 16)) || (out_f32 && !xb_aligned(out_f32, 16)) ||
        (relu_mask && !xb_aligned(relu_mask, 16)))
        return XB_EALIGN;
    if (!tma_enabled()) return XB_EINVAL;
    const int64_t K = (int64_t)n_chunks * KC;
    if (!make_tmap_box(&p.tm_a, in, C, W, in_rows, planes_a, in_plane, box_c, box_px, box_h, row_step)) return XB_EINVAL;
    if (!make_tmap(&p.tm_b, w, K, N, planes_b, K, w_plane, n_tile)) return XB_EINVAL;
    p.a_tma = p.b_tma = p.a_box = 1;
    p.mask_W = mask_W > 0 ? mask_W : out_W, p.mask_x0 = mask_W > 0 ? mask_x0 : 0;
    p.mask_ld = out_ld, p.mask_c0 = out_c0;
    p.colsum = colsum;
    p.box_w = box_w, p.box_h = box_h, p.box_hp = hp, p.box_y0 = y0, p.box_y1 = y1, p.box_rs = row_step, p.box_chunks = n_chunks;
    p.box_div_w = xb_div_make((uint32_t)box_w), p.box_div_hp = xb_div_make((uint32_t)hp);
    for (int i = 0; i < 16; ++i) p.box_c0[i] = i < n_chunks ? c0[i] : 0, p.box_w0[i] = i < n_chunks ? w0[i] : 0, p.box_r[i] = i < n_chunks ? r0[i] : 0;
    p.bias = bias;
    p.mask = (const __nv_bfloat16 *)relu_mask;
    __nv_bfloat16 *ob = (__nv_bfloat16 *)out_planes;
    p.p_out = ob ? planes_out : 0;
    for (int q = 0; q < 3; ++q) p.out[q] = (ob && q < planes_out) ? ob + q * out_plane : nullptr;
    p.out_f32 = out_f32;
    p.relu = relu;
    p.out_H = out_H, p.out_W = out_W, p.oys = oys, p.oxs = oxs, p.oy0 = oy0, p.ox0 = ox0;
    p.out_ld = out_ld, p.out_c0 = out_c0;
    p.splits = 1, p.sites_per_split = 0, p.w_ld = 0;
    p.M = (int64_t)B * hp * box_w;
    const int64_t tiles = ((int64_t)B * hp + box_h - 1) / box_h * p.n_tiles;
    return launch<false>(planes_a, planes_b, p, tiles, stream);
}

// The same GEMM with the activation tile resident in shared memory (ConvParams a_halo): stride-1 gathers over a 64-channel
// padded-row tensor - a 3x3 convolution, its data gradient, the stride phases of a strided convolution's data gradient.
extern "C" int xb_gemm_halo_tc(int planes_a, int planes_b, const void *in, int64_t in_plane, int W, int64_t in_rows, int halo_w,
                               int halo_w0, int n_sub, int n_chunks, const int16_t *dr, const int16_t *dc, const void *w,
                               int64_t w_plane, const float *bias, const void *relu_mask, int mask_W, int mask_x0, int B, int hp,
                               int y0, const int16_t *sub_y1, const int16_t *sub_x1, int N, int relu, void *out_planes,
                               int64_t out_plane, int planes_out, float *out_f32, int out_H, int out_W, int oys, int oxs,
                               const int16_t *sub_oy0, const int16_t *sub_ox0, int64_t out_ld, int out_c0, int same_cols,
                               float *colsum, void *stream) {
    if (!dr || !dc || !sub_y1 || !sub_x1 || !sub_oy0 || !sub_ox0) return XB_EINVAL;
    if (n_sub <= 0 || n_sub > 4 || n_chunks <= 0 || n_sub * n_chunks > XB_HALO_MAX_CHUNKS) return XB_ERANGE;
    if (W <= 0 || halo_w < W || halo_w > 64 || halo_w0 > 0 || halo_w0 + halo_w < W || hp <= 0 || B <= 0 || y0 < 0) return XB_EINVAL;
    if (in_rows != (int64_t)B * hp) return XB_EINVAL;
    ConvParams p;
    int8_t zero[XB_CONV_MAX_TAPS] = {0};
    // generic checks: one "tap" of 64 channels per chunk, N columns per sub-item
    const int rc = fill_params(p, planes_a, planes_b, in, in_plane, w, w_plane, B, 1, 1, 64, 1, 1, 1, 1, n_chunks, zero, zero,
                               n_sub * N, N);
    if (rc != XB_OK) return rc;
    if (!out_planes && !out_f32) return XB_EINVAL;
    if (out_planes && (planes_out < 1 || planes_out > 3)) return XB_EINVAL;
    if (out_ld % 8 != 0 || out_c0 % 8 != 0 || out_plane % 8 != 0) return XB_EALIGN;
    if ((out_planes && !xb_aligned(out_planes, 16)) || (out_f32 && !xb_aligned(out_f32, 16)) ||
        (relu_mask && !xb_aligned(relu_mask, 16)))
        return XB_EALIGN;
    if (out_ld < (int64_t)out_c0 + (same_cols ? N : n_sub * N)) return XB_EINVAL;
    if (!tma_enabled()) return XB_EINVAL;
    // shifts: positions of the haloed raster; the tile must hold [128 t + lo, 128 t + 127 + hi] for every t
    int lo = 0, hi = 0;
    for (int i = 0; i < n_sub * n_chunks; ++i) {
        // a shift is a linear offset in the raster: the pixel a VALID site (x in [0, sub_x1]) reads must stay in its own row
        const int sx1 = sub_x1[i / n_chunks];
        if (dc[i] < halo_w0 || sx1 + dc[i] > halo_w0 + halo_w - 1) return XB_ERANGE;
        const int sh = dr[i] * halo_w + dc[i];
        p.halo_shift[i] = (int16_t)sh;
        lo = sh < lo ? sh : lo, hi = sh > hi ? sh : hi;
    }
    for (int i = n_sub * n_chunks; i < XB_HALO_MAX_CHUNKS; ++i) p.halo_shift[i] = 0;
    const int halo_rows = (halo_w - 1 + TILE_M + hi - lo + halo_w - 1) / halo_w;
    if (halo_rows > 256) return XB_ERANGE;
    const uint32_t halo_plane = (((uint32_t)(halo_rows * halo_w) * 128u) + 1023u) & ~1023u;
    const uint32_t a_bytes = 2u * (uint32_t)planes_a * halo_plane, stage_bytes = (uint32_t)planes_b * xb_conv_w_plane_bytes(N);
    if (a_bytes + 2u * stage_bytes > (uint32_t)XB_K12_MAX_DYN_SMEM) return XB_ERANGE;
    int stages = (int)(((uint32_t)XB_K12_MAX_DYN_SMEM - a_bytes) / stage_bytes);
    p.stages = stages > MAX_STAGES ? MAX_STAGES : stages;
    p.dyn_smem = a_bytes + (uint32_t)p.stages * stage_bytes;
    const int64_t K = (int64_t)n_chunks * KC;
    if (!make_tmap_box(&p.tm_a, in, 64, W, in_rows, planes_a, in_plane, 64, halo_w, halo_rows, 1)) return XB_EINVAL;
    if (!make_tmap(&p.tm_b, w, K, (int64_t)n_sub * N, planes_b, K, w_plane, N)) return XB_EINVAL;
    p.a_halo = 1, p.b_tma = 1;
    p.halo_w = halo_w, p.halo_w0 = halo_w0, p.halo_rows = halo_rows, p.halo_lo = lo, p.halo_chunks = n_chunks;
    p.halo_same_cols = same_cols ? 1 : 0;
    // the 128-byte swizzle of a descriptor whose start is an arbitrary 128-byte row of a 1024-byte-aligned tile is a function
    // of the ABSOLUTE shared-memory address, exactly as TMA wrote it: the descriptors leave the matrix-base-offset field 0
    p.halo_positions = (int64_t)B * hp * halo_w;
    if (p.halo_positions + 4 * halo_w + TILE_M >= ((int64_t)1 << 31)) return XB_ERANGE;
    p.halo_div_w = xb_div_make((uint32_t)halo_w);
    p.box_hp = hp, p.box_y0 = y0, p.box_div_hp = xb_div_make((uint32_t)hp);
    for (int i = 0; i < 4; ++i) {
        const int j = i < n_sub ? i : 0;
        if (sub_y1[j] < y0 || sub_y1[j] >= hp || sub_x1[j] < 0 || sub_x1[j] >= W + 64) return XB_ERANGE;
        if ((int64_t)(sub_y1[j] - y0) * oys + sub_oy0[j] >= out_H || (int64_t)sub_x1[j] * oxs + sub_ox0[j] >= out_W || sub_oy0[j] < 0 ||
            sub_ox0[j] < 0)
            return XB_EINVAL;
        p.sub_y1[i] = sub_y1[j], p.sub_x1[i] = sub_x1[j], p.sub_oy0[i] = sub_oy0[j], p.sub_ox0[i] = sub_ox0[j];
    }
    p.bias = bias;
    p.mask = (const __nv_bfloat16 *)relu_mask;
    p.mask_W = mask_W > 0 ? mask_W : out_W, p.mask_x0 = mask_W > 0 ? mask_x0 : 0;
    p.mask_ld = out_ld, p.mask_c0 = out_c0;
    p.colsum = colsum;
    __nv_bfloat16 *ob = (__nv_bfloat16 *)out_planes;
    p.p_out = ob ? planes_out : 0;
    for (int q = 0; q < 3; ++q) p.out[q] = (ob && q < planes_out) ? ob + q * out_plane : nullptr;
    p.out_f32 = out_f32;
    p.relu = relu;
    p.out_H = out_H, p.out_W = out_W, p.oys = oys, p.oxs = oxs, p.oy0 = 0, p.ox0 = 0;
    p.out_ld = out_ld, p.out_c0 = out_c0;
    p.splits = 1, p.sites_per_split = 0, p.w_ld = 0;
    const int64_t tiles = (p.halo_positions + TILE_M - 1) / TILE_M;
    return launch<false>(planes_a, planes_b, p, tiles, stream);
}

extern "C" int xb_wgrad_gather_tc(int planes_a, int planes_b, const void *in, int64_t in_plane, const void *g, int64_t g_plane,
                                  int64_t g_ld, int B, int IH, int IW, int C, int OY, int OX, int sy, int sx, int T,
                                  const int8_t *dy, const int8_t *dx, int N, int n_tile, int splits, float *partials,
                                  void *stream) {
    ConvParams p;
    const int rc = fill_params(p, planes_a, planes_b, in, in_plane, g, g_plane, B, IH, IW, C, OY, OX, sy, sx, T, dy, dx, N, n_tile);
    if (rc != XB_OK) return rc;
    if (!partials || splits <= 0 || g_ld < N) return XB_EINVAL;
    if (!xb_aligned(partials, 16) || g_ld % 8 != 0) return XB_EALIGN;
    p.bias = nullptr, p.mask = nullptr, p.colsum = nullptr, p.out_f32 = partials, p.p_out = 0;
    for (int q = 0; q < 3; ++q) p.out[q] = nullptr;
    p.relu = 0;
    p.out_H = p.out_W = p.oys = p.oxs = 1, p.oy0 = p.ox0 = 0, p.out_ld = N, p.out_c0 = 0;
    p.w_ld = g_ld;
    const int64_t per = xb_wgrad_sites_per_split(p.M, splits);
    if (per == 0) return XB_EINVAL;     // too many splits for this many sites
    p.splits = splits, p.sites_per_split = per;
    if (tma_enabled()) {
        // output gradient [planes_b][sites][g_ld]: tiles of {64 columns, 64 sites, all planes} (one 64-column block per plane)
        if (n_tile == 64) p.b_tma = make_tmap(&p.tm_b, g, N, p.M, planes_b, g_ld, g_plane, KC) ? 1 : 0;
        // a Linear layer's input [planes_a][sites][C]: tiles of {64 columns, 64 sites, all planes}, two per 128-column tile
        if (T == 1 && IH == 1 && IW == 1 && OY == 1 && OX == 1)
            p.a_tma = make_tmap(&p.tm_a, in, C, B, planes_a, C, in_plane, KC) ? 1 : 0;
    }
    const int64_t K = (int64_t)T * C, work = (K + TILE_M - 1) / TILE_M * p.n_tiles * splits;
    return launch<true>(planes_a, planes_b, p, work, stream);
}

// Weight gradient of a convolution over padded-row tensors with BOTH operands fetched by TMA boxes (see ConvParams a_box and
// the producer): partials[s, (chunk, 64 k), n] summed over the grid rows of split s.
extern "C" int xb_wgrad_box_tc(int planes_a, int planes_b, const void *in, int64_t in_plane, int C, int W, int64_t in_rows,
                               int box_c, int box_px, int box_h, int row_step, int n_chunks, const int16_t *c0,
                               const int16_t *w0, const int16_t *r0, const void *g, int64_t g_plane, int64_t g_rows, int N,
                               int splits, float *partials, void *stream) {
    if (!c0 || !w0 || !r0 || n_chunks <= 0 || n_chunks > 16 || !partials || splits <= 0) return XB_EINVAL;
    if (box_c != 64 || box_px <= 0 || box_h <= 0 || row_step <= 0 || row_step > 8) return XB_EINVAL;
    const int box_w = box_px;
    if (box_w * box_h > KC || N % 64 != 0 || g_rows <= 0) return XB_ERANGE;
    if (!xb_aligned(partials, 16)) return XB_EALIGN;
    ConvParams p;
    int8_t zero[XB_CONV_MAX_TAPS] = {0};
    const int rc = fill_params(p, planes_a, planes_b, in, in_plane, g, g_plane, 1, 1, 1, 64, 1, 1, 1, 1, n_chunks, zero, zero, N, 64);
    if (rc != XB_OK) return rc;
    if (!tma_enabled()) return XB_EINVAL;
    if (!make_tmap_box(&p.tm_a, in, C, W, in_rows, planes_a, in_plane, box_c, box_px, box_h, row_step)) return XB_EINVAL;
    if (!make_tmap_box(&p.tm_b, g, N, box_w, g_rows, planes_b, g_plane, 64, box_w, box_h, 1)) return XB_EINVAL;
    p.a_tma = p.b_tma = p.a_box = 1;
    p.box_w = box_w, p.box_h = box_h, p.box_hp = 1, p.box_y0 = 0, p.box_y1 = 0, p.box_rs = row_step, p.box_chunks = n_chunks;
    p.box_div_w = xb_div_make((uint32_t)box_w), p.box_div_hp = xb_div_make(1u);
    for (int i = 0; i < 16; ++i) p.box_c0[i] = i < n_chunks ? c0[i] : 0, p.box_w0[i] = i < n_chunks ? w0[i] : 0, p.box_r[i] = i < n_chunks ? r0[i] : 0;
    p.bias = nullptr, p.mask = nullptr, p.colsum = nullptr, p.out_f32 = partials, p.p_out = 0;
    for (int q = 0; q < 3; ++q) p.out[q] = nullptr;
    p.relu = 0;
    p.out_H = p.out_W = p.oys = p.oxs = 1, p.oy0 = p.ox0 = 0, p.out_ld = N, p.out_c0 = 0;
    p.w_ld = N;
    // the reduction runs over the g_rows merged grid rows, cut into `splits` runs that are multiples of box_h rows
    int64_t per = (g_rows + splits - 1) / splits;
    per = (per + box_h - 1) / box_h * box_h;
    if ((int64_t)(splits - 1) * per >= g_rows) return XB_EINVAL;
    p.M = g_rows;
    p.splits = splits, p.sites_per_split = per;
    const int64_t K = (int64_t)n_chunks * KC, work = (K + TILE_M - 1) / TILE_M * p.n_tiles * splits;
    return launch<true>(planes_a, planes_b, p, work, stream);
}

// ---------------------------------------------------------------- diagnostic: raw shared-memory image of one TMA box
namespace {
__global__ void tma_probe_kernel(const __grid_constant__ CUtensorMap tm, int c0, int c1, int c2, int c3, int rs, uint32_t bytes,
                                 uint8_t *out, uint32_t out_bytes) {
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar;
    for (uint32_t i = threadIdx.x; i < out_bytes; i += blockDim.x) smem[i] = 0xEE;
    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
        mbar_fence_init();
    }
    fence_proxy_async();
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&bar, bytes);
        tma_load_box(smem_u32(smem), &tm, c0, c1, c2, rs, c3, &bar);
    }
    mbar_wait(&bar, 0);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < out_bytes; i += blockDim.x) out[i] = smem[i];
}
}  // namespace

// test hook: loads ONE box of the 4-D map make_tmap_box would build and returns the first out_bytes of shared memory (0xEE =
// never written), so that the layout assumptions of the box mode can be checked byte for byte (tests/test_gpu_tc_conv.py)
// XB_K12_TIMING=1 diagnostics: the role timing table of the last K12 launch (see xb_k12_timing), copied to a HOST array
extern "C" int xb_debug_k12_timing(unsigned long long *out_host, int n_ctas) {
    if (!out_host || n_ctas <= 0 || n_ctas > 160) return XB_EINVAL;
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpyFromSymbol(out_host, xb_k12_timing, sizeof(unsigned long long) * 12 * n_ctas);
    return e == cudaSuccess ? XB_OK : (int)e;
}

extern "C" int xb_debug_tma_box(const void *in, int64_t in_plane, int planes, int C, int W, int64_t rows, int box_c, int box_px,
                                int box_h, int row_step, int c0, int c1, int c2, int c3, uint32_t expect_bytes, void *out,
                                uint32_t out_bytes, void *stream) {
    CUtensorMap tm;
    if (!make_tmap_box(&tm, in, C, W, rows, planes, in_plane, box_c, box_px, box_h, row_step)) return XB_EINVAL;
    if (out_bytes > 64 * 1024) return XB_ERANGE;
    cudaFuncSetAttribute(tma_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    tma_probe_kernel<<<1, 256, 64 * 1024, (cudaStream_t)stream>>>(tm, c0, c1, c2, c3, row_step, expect_bytes, (uint8_t *)out, out_bytes);
    return xb_launch_status();
}

extern "C" int xb_wgrad_reduce(float *partials, int splits, int N, int C, int KH, int KW, float scale, float *dw, int accumulate,
                               void *stream) {
    if (!partials || !dw || splits <= 0 || N <= 0 || C <= 0 || KH <= 0 || KW <= 0) return XB_EINVAL;
    const int64_t total = (int64_t)N * C * KH * KW;
    auto lanes_for = [&](int n_splits, int64_t groups) {
        int lanes = 1;
        while (lanes < 8 && lanes * 2 <= n_splits && total / (256 / lanes) * groups < (int64_t)xb_sm_count() * 16) lanes *= 2;
        return lanes;
    };
    int step = 1;
    if (splits > 256) {                     // fold groups of consecutive splits in place first (see wgrad_fold_kernel)
        const int group = (splits + 127) / 128, groups = (splits + group - 1) / group;
        const int lanes = lanes_for(group, groups);
        const int64_t E = 256 / lanes, bx = (total + E - 1) / E;
        if (bx > 0x7fffffff || groups > 65535) return XB_ERANGE;
        wgrad_fold_kernel<<<dim3((unsigned)bx, (unsigned)groups), 256, 0, (cudaStream_t)stream>>>(partials, splits, group, lanes, total);
        step = group;
    }
    // (worth it only for a big weight with few splits: a block walks its 32 x 2 x HW tile once per split)
    if (xb_pack_tiled(3, N, C, KH * KW) && KH * KW <= 128 && (N / 32) * (C / 2) >= 128 && (splits + step - 1) / step <= 16) {
        wgrad_reduce_tiled_kernel<<<(unsigned)((N / 32) * (C / 2)), 256, 0, (cudaStream_t)stream>>>(partials, splits, step, N, C, KH * KW,
                                                                                            scale, dw, accumulate);
        return xb_launch_status();
    }
    const int lanes = lanes_for((splits + step - 1) / step, 1);
    const int64_t E = 256 / lanes;
    if ((total + E - 1) / E > 0x7fffffff) return XB_ERANGE;
    wgrad_reduce_kernel<<<(int)((total + E - 1) / E), 256, 0, (cudaStream_t)stream>>>(partials, splits, step, lanes, N, C, KH, KW, scale, dw,
                                                                                  accumulate);
    return xb_launch_status();
}

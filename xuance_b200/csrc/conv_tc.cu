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
//                          pa, the A fragment is read ONCE into registers (ldmatrix) and wgmmas of 64 / 32 columns multiply
//                          it with the first PB - pa B planes (adjacent in the stage = ONE operand of (PB - pa) * N rows, read
//                          from shared memory) into the register accumulator blocks of groups pa .. PB-1; the wgmmas of a
//                          chunk form one group, and its stage is released when that group has retired.
//   Registers: setmaxnreg moves them from the producer warpgroup to the consumers (PROD_REGS / CONS_REGS).
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
// exit to xb_k12_timing[b][..]: 0 consumer total, 1 consumer wait full (operands), 2 consumer wgmma_wait (MMAs in flight),
// 3 consumer wait a_full (halo tile), 4 producer total, 5 producer wait empty (ring), 6 producer wait a_empty, 7 consumer
// epilogue (last stage released .. column sums stored) (tools/k12_timing.py); the other slots are unused
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
    // conv_tc_kernel_wgrad_win: window slots per chunk, slot pitch in bytes, KH input rows and win_w units per slot;
    // conv_tc_kernel_wgrad_pairs: the same with one input row and win_w pixel pairs per slot and plane
    int win_rows, win_kh, win_w;
    uint32_t win_slot;
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
// TMA: one 5-D box at coordinates {c0 .. c4} -> shared memory, completion bytes on an mbarrier
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap *tm, int c0, int c1, int c2, int c3, int c4, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
        ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(smem_u32(bar))
        : "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// bulk copy shared -> global (the copy engine, no per-lane stores), completion tracked per issuing thread in bulk groups
__device__ __forceinline__ void bulk_store(void *dst, uint32_t src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every bulk group this thread committed has finished READING shared memory (its source may be overwritten)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// x = hi + mid + lo, three bf16 values: 24 mantissa bits, |x - hi - mid - lo| <= 2^-24 |x|
__device__ __forceinline__ void split3_bf16(float x, __nv_bfloat16 &hi, __nv_bfloat16 &mid, __nv_bfloat16 &lo) {
    hi = __float2bfloat16_rn(x);
    const float r1 = x - __bfloat162float(hi);
    mid = __float2bfloat16_rn(r1);
    lo = __float2bfloat16_rn(r1 - __bfloat162float(mid));
}

// A plane (its fragment in registers) x the first PB - pa B planes for one K step: the accumulator blocks pa*NC .. PB*NC-1
// (32 columns each).  Block j reads B rows 32 (j - pa*NC) .. +31 of the stage: 4096 bytes per block in every operand layout
// the kernel uses (128 bytes per row or per MN index).  In-flight wgmmas are ordered on their accumulator registers only
// when they have the same shape and register set, so every block is always written by the same instruction form: pairs
// (2i, 2i+1) as one n64 wgmma when NC is even (then every plane's range starts at an even block), single n32 wgmmas when NC
// is odd.
template <int TB, int PB, int NC, int PA_>
__device__ __forceinline__ void mma_plane(float (&acc)[PB * NC][16], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    constexpr int J0 = PA_ * NC, J1 = PB * NC, STEP = NC % 2 == 0 ? 2 : 1;
#pragma unroll
    for (int j = J0; j < J1; j += STEP) {
        const uint64_t b = db + (uint64_t)(((j - J0) * 4096) >> 4);
        if (STEP == 2) wgmma_rs_n64<TB>(acc[j], acc[j + 1 < J1 ? j + 1 : j], a, b, scale_d);
        else wgmma_rs_n32<TB>(acc[j], a, b, scale_d);
    }
}

// role timing: the low 32 bits of the SM clock (differences and sums of waits stay far below 2^32 cycles in one launch;
// 32-bit sums keep the consumers' register budget)
__device__ __forceinline__ uint32_t clock32() {
    uint32_t c;
    asm volatile("mov.u32 %0, %%clock;" : "=r"(c));
    return c;
}
// wgmma_wait<N>, its cycles added to `cycles` when the role timing is on
template <int N>
__device__ __forceinline__ void timed_wgmma_wait(bool timing, uint32_t &cycles) {
    if (timing) {
        const uint32_t t0 = clock32();
        wgmma_wait<N>();
        cycles += clock32() - t0;
    } else {
        wgmma_wait<N>();
    }
}

// register split between the roles (setmaxnreg): 384 threads at the 168 registers one CTA per SM allows = 64512 per CTA;
// the producer warpgroup gives back to PROD_REGS and the consumer warpgroups, which hold the accumulators and the double
// buffered A fragments, take CONS_REGS: 2 * 128 * CONS_REGS + 128 * PROD_REGS must not exceed 128 * 3 * 168, or the
// consumers' setmaxnreg.inc would wait for registers that never come free
constexpr int LAUNCH_REGS = 168, PROD_REGS = 104, CONS_REGS = 200;
static_assert(2 * CONS_REGS + PROD_REGS <= 3 * LAUNCH_REGS && THREADS == 3 * 128, "register split");

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
    uint32_t t_wait[5] = {0, 0, 0, 0, 0};                   // role timing: slots 0-2 barrier waits, 3 wgmma_wait, 4 epilogue
    // role timing: the two reporting threads park their start clock in their total slot until kernel exit (not in a
    // register that would stay live across the whole main loop)
    if (p.timing && blockIdx.x < 160 && (tid == 0 || tid == CONS_WARPS * 32)) xb_k12_timing[blockIdx.x][tid == 0 ? 0 : 4] = clock64();
    auto timed_wait = [&](uint64_t *bar, uint32_t parity, int slot) {
        if (p.timing) {
            const uint32_t t0 = clock32();
            mbar_wait(bar, parity);
            t_wait[slot] += clock32() - t0;
        } else {
            mbar_wait(bar, parity);
        }
    };
    if ((p.a_tma || p.b_tma) && (smem_base & 1023u)) __trap();     // the 128-byte swizzle pattern repeats every 1024 B

    if (warp >= CONS_WARPS) {
        // ------------------------------------------------------------------ producers (128 threads)
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
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
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONS_REGS));
        //  A (read into registers with ldmatrix, one x4 per K step of 16 and plane; warpgroup wg reads rows 64 wg .. +63):
        //     halo     128-byte swizzle K-major window of the resident tile, planes halo_plane apart
        //     cp.async no-swizzle canonical layout (conv_index.h): K-major forward, MN-major weight gradient, K step = two
        //              core matrices = 256 B, planes a_plane apart
        //     TMA      128-byte swizzle.  K-major: rows of 128 B, K step 32 B.  MN-major (weight gradient): two blocks of 64
        //              columns, each [planes][64 sites][128 B]: plane stride a_plane/2, block stride PA*a_plane/2, K step 2048 B
        //  B: the first (PB - pa) planes, adjacent in the stage, are ONE operand of (PB - pa) * N rows (same three layouts;
        //     MN-major: one 64-column block per plane, blocks w_plane apart); descriptor = per-launch template (layout, LBO,
        //     SBO) + start address in 16-byte units
        const int wg = warp >> 2;
        uint64_t b_tmpl;
        uint32_t b_ks;                                       // per K step of 16, in 16-byte units
        if (!p.b_tma) b_tmpl = make_desc(0, KC), b_ks = 256 >> 4;
        else if (!WGRAD) b_tmpl = make_desc_sw128(0, 16, 1024), b_ks = 32 >> 4;
        else b_tmpl = make_desc_sw128(0, w_plane, 1024), b_ks = 2048 >> 4;
        // this lane's ldmatrix row: matrix mi = lane / 8 of the x4 holds rows (m) + 8 (mi & 1), K columns + 8 (mi >> 1) of
        // the warp's 16 x 16 fragment; lane & 7 is its row of that 8 x 8 matrix (an m row K-major, a k row MN-major)
        const int mi = lane >> 3, lr = lane & 7, m_l = 16 * (warp & 3) + 8 * (mi & 1);
        // a_lane: byte offset of the lane's 16-byte row at K step 0 from the stage's A base, a_ks: per K step (linear
        // layouts), a_pl: per plane (multiples of 1024 B: the swizzle phase is the same for every plane)
        const bool a_sw_k = !WGRAD && (halo || p.a_tma);     // 128-byte swizzle, K-major: the K step is an XOR on the 16-byte unit
        uint32_t a_lane, a_ks, a_pl;
        if (!WGRAD) {
            if (a_sw_k) a_lane = (uint32_t)wg * 8192u + (uint32_t)(m_l + lr) * 128u, a_ks = 0, a_pl = halo ? halo_plane : a_plane;
            else a_lane = (uint32_t)wg * 8192u + (uint32_t)((m_l + lr) >> 3) * 1024u + (uint32_t)(mi >> 1) * 128u + lr * 16u,
                 a_ks = 256, a_pl = a_plane;
        } else if (p.a_tma) {
            a_lane = (uint32_t)wg * PA * (a_plane / 2) + (uint32_t)(8 * (mi >> 1) + lr) * 128u + (uint32_t)(((m_l >> 3) ^ lr) << 4);
            a_ks = 2048, a_pl = a_plane / 2;
        } else {
            a_lane = (uint32_t)wg * 8192u + (uint32_t)(m_l >> 3) * 1024u + (uint32_t)(mi >> 1) * 128u + lr * 16u;
            a_ks = 256, a_pl = a_plane;
        }
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
            uint32_t af[KC / 16][PA][4];                      // A fragments of a chunk, one register set per K step and plane
            for (int kc = 0; kc < n_chunks; ++kc) {
                const int stage = (int)(it % (uint32_t)S);
                timed_wait(&full_bar[stage], (it / (uint32_t)S) & 1u, 0);
                fence_proxy_async();       // the stage was written by cp.async (generic proxy); the MMA reads it through the async proxy
                const uint32_t base = smem_base + ring_off + (uint32_t)stage * stage_bytes;
                const uint32_t w_addr = base + (halo ? 0u : PA * a_plane);
                const uint32_t a_row = a_lane + (halo ? halo_base + (uint32_t)(halo_s0 + p.halo_shift[sub * p.halo_chunks + kc]) * 128u : base);
                // the 128-byte swizzle XORs the 16-byte unit with bits 7-9 of the ABSOLUTE address, as TMA wrote it (a halo
                // window starts at any 128-byte row of its 1024-byte-aligned tile)
                const uint32_t a_sw = (a_row >> 7) & 7u;
                // start addresses stay below 2^18 bytes: adding 16-byte units to the template never carries out of the field
                const uint64_t b0 = b_tmpl + (uint64_t)(w_addr >> 4);
                // every fragment of the chunk is loaded while no wgmma is in flight: registers a pending wgmma reads are
                // never redefined (otherwise ptxas serialises every wgmma of the kernel)
#pragma unroll
                for (int ks = 0; ks < KC / 16; ++ks) {
                    const uint32_t a_addr = a_sw_k ? a_row + (((uint32_t)(2 * ks + (mi >> 1))) ^ a_sw) * 16u : a_row + (uint32_t)ks * a_ks;
#pragma unroll
                    for (int q = 0; q < PA; ++q) ldmatrix_x4<TR>(af[ks][q], a_addr + (uint32_t)q * a_pl);
                }
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < KC / 16; ++ks) {
                    // A plane pa x B planes 0 .. PB-1-pa -> accumulator groups pa .. PB-1.
                    // pa = 0 covers every group, so its first instruction of a work item (scale_d = 0) initialises them all.
                    const uint64_t db = b0 + (uint64_t)(ks * b_ks);
                    mma_plane<TR, PB, NC, 0>(acc, af[ks][0], db, scale_d);
                    if (PA > 1) mma_plane<TR, PB, NC, (PA > 1 ? 1 : 0)>(acc, af[ks][PA > 1 ? 1 : 0], db, 1u);
                    if (PA > 2) mma_plane<TR, PB, NC, (PA > 2 ? 2 : 0)>(acc, af[ks][PA > 2 ? 2 : 0], db, 1u);
                    scale_d = 1;
                }
                wgmma_commit();
                timed_wgmma_wait<0>(p.timing, t_wait[3]);
                // every wgmma that read the stage has retired: it is free
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[stage]);
                ++it;
            }
            const uint32_t t_epi = p.timing ? clock32() : 0u;
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
                // the ReLU mask of these 32 columns, all its words loaded before any store (the mask and the outputs may alias
                // as far as the compiler knows: a load issued after a store would wait out its whole latency, once per
                // 8-column block and row) and kept as one bit per element, bit 4 (2 i + h) + e; bf16 > 0 <=> sign bit clear
                // and not (+)zero
                uint32_t keep = 0u;
                if (!WGRAD && p.mask) {
                    uint32_t mw[4][2];
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            mw[i][h] = live[h] ? *reinterpret_cast<const uint32_t *>(p.mask + mrow[h] + 32 * cc + 8 * i + cq) : 0u;
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const uint32_t lo16 = mw[i][h] & 0xffffu, hi16 = mw[i][h] >> 16;
                            keep |= (uint32_t)(lo16 != 0u && lo16 < 0x8000u) << (4 * (2 * i + h));
                            keep |= (uint32_t)(hi16 != 0u && hi16 < 0x8000u) << (4 * (2 * i + h) + 1);
                        }
                }
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
                                if (p.mask && !((keep >> (4 * (2 * i + h) + e)) & 1u)) v[e] = 0.f;
                            }
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
            if (p.timing) t_wait[4] += clock32() - t_epi;
          }
          if (halo) {
              __syncwarp();                                   // every MMA of this tile has retired (wait above)
              if (lane == 0) mbar_arrive(&a_empty[tile_it & 1u]);
              ++tile_it;
          }
        }
    }
    if (p.timing && blockIdx.x < 160) {
        const unsigned long long now = clock64();
        unsigned long long *o = xb_k12_timing[blockIdx.x];
        if (tid == 0) o[0] = now - o[0], o[1] = t_wait[0], o[2] = t_wait[3], o[3] = t_wait[2], o[7] = t_wait[4];
        if (tid == CONS_WARPS * 32) o[4] = now - o[4], o[5] = t_wait[0], o[6] = t_wait[1];
    }
}

// The weight gradient of a raw-pixel first layer (one A plane, C = 8, a full tap rectangle, N = 32, K <= 256; selected by
// xb_wgrad_gather_tc) with both operands by TMA: work item = one split, ALL K rows, so every site's patches and output
// gradient are loaded once instead of once per 128-row tile.  Per chunk of 64 sites one elected producer thread loads
//   * the output gradient: one box {32 columns, 64 sites, PB planes}, 64-byte swizzle ([plane][site][64 B]);
//   * the input window: win_rows boxes of KH rows x win_w 16-byte units (conv_index.h, xb_win_*), no swizzle;
// and the consumer warps read their MN-major A fragments with ldmatrix.trans straight from the window (the 16 bytes of a
// fragment row are one tap unit of one site).  Warpgroup wg owns the m64 row blocks wg and wg + 2 (rows 128 r + 64 wg ..),
// the rows of the gathered path's tile r, and issues per K step and row block the same n32 wgmmas on the same fragments,
// B planes and accumulators in the same order, so the partials are bit for bit those of conv_tc_kernel<true, 1, PB, 1>.
template <int PB>
__global__ void __launch_bounds__(THREADS, 1) conv_tc_kernel_wgrad_win(const __grid_constant__ ConvParams p) {
    constexpr int RB = 2;                                    // m64 row blocks per consumer warpgroup
    constexpr uint32_t G_BYTES = PB * 32 * XB_CONV_KC * 2;   // output-gradient box: 4096 B per plane
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t full_bar[MAX_STAGES], empty_bar[MAX_STAGES];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const XbConvGeom &g = p.g;
    const int K = g.T * g.C, S = p.stages;
    const uint32_t stage_bytes = (G_BYTES + (uint32_t)p.win_rows * p.win_slot + 1023u) & ~1023u;   // as wgrad_win_setup
    auto chunks_of = [&](int64_t sp) -> int {
        const int64_t s0 = sp * p.sites_per_split, cnt = (p.M - s0) < p.sites_per_split ? (p.M - s0) : p.sites_per_split;
        return (int)((cnt + KC - 1) / KC);
    };
    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], CONS_WARPS);
        }
        mbar_fence_init();
    }
    __syncthreads();
    const uint32_t smem_base = smem_u32(smem);
    uint32_t t_wait[5] = {0, 0, 0, 0, 0};                   // role timing, slots as in conv_tc_kernel
    if (p.timing && blockIdx.x < 160 && (tid == 0 || tid == CONS_WARPS * 32)) xb_k12_timing[blockIdx.x][tid == 0 ? 0 : 4] = clock64();
    auto timed_wait = [&](uint64_t *bar, uint32_t parity, int slot) {
        if (p.timing) {
            const uint32_t t0 = clock32();
            mbar_wait(bar, parity);
            t_wait[slot] += clock32() - t0;
        } else {
            mbar_wait(bar, parity);
        }
    };

    if (warp >= CONS_WARPS) {
        // ------------------------------------------------------------------ producer: one thread issues every copy
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
        if (tid == CONS_WARPS * 32) {
            const uint32_t bytes = G_BYTES + (uint32_t)(p.win_rows * p.win_kh * p.win_w * 16);
            uint32_t it = 0;
            for (int64_t sp = blockIdx.x; sp < p.splits; sp += gridDim.x) {
                const int n_chunks = chunks_of(sp);
                for (int kc = 0; kc < n_chunks; ++kc, ++it) {
                    const int stage = (int)(it % (uint32_t)S);
                    timed_wait(&empty_bar[stage], ((it / (uint32_t)S) & 1u) ^ 1u, 0);
                    const uint32_t base = smem_base + (uint32_t)stage * stage_bytes;
                    const int64_t site0 = sp * p.sites_per_split + (int64_t)kc * KC;
                    mbar_expect_tx(&full_bar[stage], bytes);
                    tma_load_3d(base, &p.tm_b, 0, (int)site0, 0, &full_bar[stage]);            // G[site, n], sites >= M zero
                    const int64_t R0 = xb_div((uint32_t)site0, g.div_ox);      // first grid row of the chunk
                    for (int j = 0; j < p.win_rows; ++j) {
                        int b, iy0;
                        xb_win_box(g, R0 + j, b, iy0);
                        // 8-byte elements: unit u is elements 2u, 2u + 1
                        tma_load_3d(base + G_BYTES + (uint32_t)j * p.win_slot, &p.tm_a, 2 * g.dx[0], iy0, b, &full_bar[stage]);
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ consumers: wgmma issue + epilogue
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONS_REGS));
        const int wg = warp >> 2;
        // B: MN-major, 64-byte swizzle, 8-site groups of 512 B (SBO), K step of 16 sites = 1024 B, planes 4096 B apart
        const uint64_t b_tmpl = make_desc_sw64(0, 0, 512);
        // this lane's ldmatrix row (see conv_tc_kernel): k row = site 8 (mi >> 1) + lr of the K step, m rows = the 8 K-unit
        // columns from m_l of the warp's 16 x 16 fragment
        const int mi = lane >> 3, lr = lane & 7, m_l = 16 * (warp & 3) + 8 * (mi & 1);
        uint32_t tap_off[RB];
#pragma unroll
        for (int r = 0; r < RB; ++r) tap_off[r] = xb_win_tap_off(g, 128 * r + 64 * wg + m_l, p.win_w);
        const int rbase = 64 * wg + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
        float acc[RB][PB][16];
        uint32_t it = 0;
        for (int64_t sp = blockIdx.x; sp < p.splits; sp += gridDim.x) {
            const int n_chunks = chunks_of(sp);
            uint32_t scale_d = 0;
            uint32_t af[KC / 16][RB][4];
            for (int kc = 0; kc < n_chunks; ++kc, ++it) {
                const int stage = (int)(it % (uint32_t)S);
                const uint32_t base = smem_base + (uint32_t)stage * stage_bytes;
                const int64_t site0 = sp * p.sites_per_split + (int64_t)kc * KC;
                const int64_t R0 = xb_div((uint32_t)site0, g.div_ox);      // first grid row of the chunk
                uint32_t site_off[KC / 16];
#pragma unroll
                for (int ks = 0; ks < KC / 16; ++ks) site_off[ks] = xb_win_site_off(g, site0 + 16 * ks + 8 * (mi >> 1) + lr, R0, p.win_slot);
                timed_wait(&full_bar[stage], (it / (uint32_t)S) & 1u, 0);
                const uint32_t win = base + G_BYTES;
                // every fragment of the chunk is loaded while no wgmma is in flight (see conv_tc_kernel)
#pragma unroll
                for (int ks = 0; ks < KC / 16; ++ks)
#pragma unroll
                    for (int r = 0; r < RB; ++r) ldmatrix_x4<1>(af[ks][r], win + site_off[ks] + tap_off[r]);
                wgmma_fence();
                const uint64_t b0 = b_tmpl + (uint64_t)(base >> 4);
#pragma unroll
                for (int ks = 0; ks < KC / 16; ++ks) {
#pragma unroll
                    for (int r = 0; r < RB; ++r)
#pragma unroll
                        for (int q = 0; q < PB; ++q)
                            wgmma_rs_n32<1>(acc[r][q], af[ks][r], b0 + (uint64_t)((ks * 1024 + q * 4096) >> 4), scale_d);
                    scale_d = 1;
                }
                wgmma_commit();
                timed_wgmma_wait<0>(p.timing, t_wait[3]);
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[stage]);
            }
            const uint32_t t_epi = p.timing ? clock32() : 0u;
            // ---- epilogue: partials [splits, K, 32], rows 128 r + rbase (+ 8), accumulator groups added smallest first
#pragma unroll
            for (int r = 0; r < RB; ++r)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int kcol = 128 * r + rbase + 8 * h;
                    if (kcol >= K) continue;
                    float *row = p.out_f32 + (sp * K + kcol) * 32;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        float v[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            v[e] = acc[r][PB - 1][4 * i + 2 * h + e];
#pragma unroll
                            for (int gq = PB - 2; gq >= 0; --gq) v[e] += acc[r][gq][4 * i + 2 * h + e];
                        }
                        *reinterpret_cast<float2 *>(row + 8 * i + cq) = make_float2(v[0], v[1]);
                    }
                }
            if (p.timing) t_wait[4] += clock32() - t_epi;
        }
    }
    if (p.timing && blockIdx.x < 160) {
        const unsigned long long now = clock64();
        unsigned long long *o = xb_k12_timing[blockIdx.x];
        if (tid == 0) o[0] = now - o[0], o[1] = t_wait[0], o[2] = t_wait[3], o[3] = 0, o[7] = t_wait[4];
        if (tid == CONS_WARPS * 32) o[4] = now - o[4], o[5] = t_wait[0], o[6] = 0;
    }
}

// The weight gradient of a stride-2 layer over a 32-channel activation read as pixel pairs (three planes each side, C = 32,
// a KH x 4 tap rectangle, N = n_tile = 64; selected by xb_wgrad_gather_tc) with both operands by TMA.  Work items, chunks
// and wgmmas are the gathered path's: item = (split, 128-row K tile mt) split-major, so the K tiles of a split run on
// neighbouring CTAs at the same time and share their loads in L2.  Per chunk of 64 sites one elected producer thread loads
//   * the output gradient: one box {64 columns, 64 sites, 3 planes}, 128-byte swizzle (the gathered path's b_tma box);
//   * the input window: win_rows boxes {64 channels, win_w pairs, input row sy * y + dy[4 mt] of image b, 3 planes}, 128-byte
//     swizzle, one per grid row (b, y) the chunk can touch (conv_index.h, xb_pwin_*);
// and the consumer warps read their MN-major A fragments with ldmatrix.trans straight from the window (a fragment row is 8
// channels of one site and pair; 8 consecutive sites are 8 consecutive 128-byte pair rows, which the swizzle spreads over
// all banks).  Each warpgroup issues the gathered path's n64 wgmmas on the same fragments, B planes and accumulators in
// the same order, so the partials are bit for bit those of conv_tc_kernel<true, 3, 3, 2>.
__global__ void __launch_bounds__(THREADS, 1) conv_tc_kernel_wgrad_pairs(const __grid_constant__ ConvParams p) {
    constexpr int PA = 3, PB = 3, NC = 2, N = 32 * NC;
    constexpr uint32_t G_BYTES = PB * N * KC * 2;            // output-gradient box: 8192 B per plane
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t full_bar[MAX_STAGES], empty_bar[MAX_STAGES];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const XbConvGeom &g = p.g;
    const int K = g.T * g.C, S = p.stages, m_tiles = K / TILE_M;
    const int64_t n_work = (int64_t)p.splits * m_tiles;
    const uint32_t stage_bytes = G_BYTES + (uint32_t)p.win_rows * p.win_slot;     // as wgrad_pairs_setup
    const uint32_t pair_plane = (uint32_t)p.win_w * 128u;                          // one plane of a window slot
    auto chunks_of = [&](int64_t sp) -> int {
        const int64_t s0 = sp * p.sites_per_split, cnt = (p.M - s0) < p.sites_per_split ? (p.M - s0) : p.sites_per_split;
        return (int)((cnt + KC - 1) / KC);
    };
    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], CONS_WARPS);
        }
        mbar_fence_init();
    }
    __syncthreads();
    const uint32_t smem_base = smem_u32(smem);
    if (smem_base & 1023u) __trap();                         // the 128-byte swizzle pattern repeats every 1024 B
    uint32_t t_wait[5] = {0, 0, 0, 0, 0};                   // role timing, slots as in conv_tc_kernel
    if (p.timing && blockIdx.x < 160 && (tid == 0 || tid == CONS_WARPS * 32)) xb_k12_timing[blockIdx.x][tid == 0 ? 0 : 4] = clock64();
    auto timed_wait = [&](uint64_t *bar, uint32_t parity, int slot) {
        if (p.timing) {
            const uint32_t t0 = clock32();
            mbar_wait(bar, parity);
            t_wait[slot] += clock32() - t0;
        } else {
            mbar_wait(bar, parity);
        }
    };

    if (warp >= CONS_WARPS) {
        // ------------------------------------------------------------------ producer: one thread issues every copy
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
        if (tid == CONS_WARPS * 32) {
            const uint32_t bytes = G_BYTES + (uint32_t)p.win_rows * (uint32_t)PA * pair_plane;
            const int p0 = g.dx[0] / 2;                      // first pair of a window row (dx[0] even)
            uint32_t it = 0;
            for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x) {
                const int64_t sp = w / m_tiles;
                const int mt = (int)(w - sp * m_tiles);
                const int n_chunks = chunks_of(sp);
                for (int kc = 0; kc < n_chunks; ++kc, ++it) {
                    const int stage = (int)(it % (uint32_t)S);
                    timed_wait(&empty_bar[stage], ((it / (uint32_t)S) & 1u) ^ 1u, 0);
                    const uint32_t base = smem_base + (uint32_t)stage * stage_bytes;
                    const int64_t site0 = sp * p.sites_per_split + (int64_t)kc * KC;
                    mbar_expect_tx(&full_bar[stage], bytes);
                    tma_load_3d(base, &p.tm_b, 0, (int)site0, 0, &full_bar[stage]);            // G[site, n], sites >= M zero
                    const int64_t R0 = xb_div((uint32_t)site0, g.div_ox);      // first grid row of the chunk
                    for (int j = 0; j < p.win_rows; ++j) {
                        int b, iy;
                        xb_pwin_box(g, R0 + j, mt, b, iy);
                        tma_load_5d(base + G_BYTES + (uint32_t)j * p.win_slot, &p.tm_a, 0, p0, iy, b, 0, &full_bar[stage]);
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ consumers: wgmma issue + epilogue
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONS_REGS));
        const int wg = warp >> 2;
        // B as in conv_tc_kernel's weight gradient with b_tma: MN-major, 128-byte swizzle, planes w_plane = 8192 B apart,
        // K step of 16 sites = 2048 B
        const uint64_t b_tmpl = make_desc_sw128(0, xb_conv_w_plane_bytes(N), 1024);
        // this lane's ldmatrix row (see conv_tc_kernel): k row = site 8 (mi >> 1) + lr of the K step, m rows = the 8 K rows
        // from 64 wg + m_l of the tile
        const int mi = lane >> 3, lr = lane & 7, m_l = 16 * (warp & 3) + 8 * (mi & 1);
        const uint32_t tap_off = xb_pwin_tap_off(g, 64 * wg + m_l);
        const int rbase = 64 * wg + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
        float acc[PB * NC][16];
        uint32_t it = 0;
        for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x) {
            const int64_t sp = w / m_tiles;
            const int mt = (int)(w - sp * m_tiles);
            const int n_chunks = chunks_of(sp);
            uint32_t scale_d = 0;
            uint32_t af[KC / 16][PA][4];
            for (int kc = 0; kc < n_chunks; ++kc, ++it) {
                const int stage = (int)(it % (uint32_t)S);
                const uint32_t base = smem_base + (uint32_t)stage * stage_bytes;
                const int64_t site0 = sp * p.sites_per_split + (int64_t)kc * KC;
                const int64_t R0 = xb_div((uint32_t)site0, g.div_ox);      // first grid row of the chunk
                const uint32_t win = base + G_BYTES + tap_off;
                uint32_t row[KC / 16];
#pragma unroll
                for (int ks = 0; ks < KC / 16; ++ks) row[ks] = win + xb_pwin_site_off(g, site0 + 16 * ks + 8 * (mi >> 1) + lr, R0, p.win_slot);
                timed_wait(&full_bar[stage], (it / (uint32_t)S) & 1u, 0);
                // every fragment of the chunk is loaded while no wgmma is in flight (see conv_tc_kernel)
#pragma unroll
                for (int ks = 0; ks < KC / 16; ++ks)
#pragma unroll
                    for (int q = 0; q < PA; ++q) ldmatrix_x4<1>(af[ks][q], xb_sw128(row[ks] + (uint32_t)q * pair_plane));
                wgmma_fence();
                const uint64_t b0 = b_tmpl + (uint64_t)(base >> 4);
#pragma unroll
                for (int ks = 0; ks < KC / 16; ++ks) {
                    const uint64_t db = b0 + (uint64_t)(ks * (2048 >> 4));
                    mma_plane<1, PB, NC, 0>(acc, af[ks][0], db, scale_d);
                    mma_plane<1, PB, NC, 1>(acc, af[ks][1], db, 1u);
                    mma_plane<1, PB, NC, 2>(acc, af[ks][2], db, 1u);
                    scale_d = 1;
                }
                wgmma_commit();
                timed_wgmma_wait<0>(p.timing, t_wait[3]);
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[stage]);
            }
            const uint32_t t_epi = p.timing ? clock32() : 0u;
            // ---- epilogue: partials [splits, K, 64], rows 128 mt + rbase (+ 8), accumulator groups added smallest first
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float *row = p.out_f32 + (sp * K + 128 * mt + rbase + 8 * h) * N;
#pragma unroll
                for (int cc = 0; cc < NC; ++cc)
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        float v[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            v[e] = acc[(PB - 1) * NC + cc][4 * i + 2 * h + e];
#pragma unroll
                            for (int gq = PB - 2; gq >= 0; --gq) v[e] += acc[gq * NC + cc][4 * i + 2 * h + e];
                        }
                        *reinterpret_cast<float2 *>(row + 32 * cc + 8 * i + cq) = make_float2(v[0], v[1]);
                    }
            }
            if (p.timing) t_wait[4] += clock32() - t_epi;
        }
    }
    if (p.timing && blockIdx.x < 160) {
        const unsigned long long now = clock64();
        unsigned long long *o = xb_k12_timing[blockIdx.x];
        if (tid == 0) o[0] = now - o[0], o[1] = t_wait[0], o[2] = t_wait[3], o[3] = 0, o[7] = t_wait[4];
        if (tid == CONS_WARPS * 32) o[4] = now - o[4], o[5] = t_wait[0], o[6] = 0;
    }
}

// The forward of a raw-pixel first layer (one A plane, C = 8, a full tap rectangle, K = 256, N = 32, bf16 plane outputs
// whose sites are 64-byte rows, no mask / column sums; selected by xb_gemm_gather_tc) with every transfer on the copy
// engines.  Work items are the gathered path's: 128 consecutive sites, rows 0-63 / 64-127 for the two consumer warpgroups.
//   * weights: RESIDENT, loaded once per CTA by TMA (the gathered path's b_tma boxes: per 64-deep chunk {64 k, 32 rows, PB
//     planes}, 128-byte swizzle);
//   * input: per item one window (conv_index.h, xb_win_*) of xb_win_rows(g, 128) boxes of KH rows x win_w units, zero fill
//     for padding and past the last image; two stages.  An item reads all K from it, so it needs no per-chunk loads;
//   * outputs: the consumers write the split bf16 planes into a staging tile [plane][128 sites][64 B] and, after a named
//     barrier, lane j of warp 0 copies the run of the item's sites in grid row R0 + j (consecutive real pixels, contiguous
//     in every plane of the output) with one cp.async.bulk per plane.  Two staging tiles: a tile is rewritten only after the
//     copies that read it have been waited for (wait_group.read before the barrier of the next item).
// The consumers read K-major A fragments with ldmatrix at xb_win_site_off + xb_win_tap_off and issue per K step the
// gathered path's n32 wgmmas on the same fragments, B planes and accumulators in the same order, and the epilogue adds the
// groups, bias and ReLU as it does: the outputs are bit for bit those of conv_tc_kernel<false, 1, PB, 1>.
template <int PB>
__global__ void __launch_bounds__(THREADS, 1) conv_tc_kernel_fwd_win(const __grid_constant__ ConvParams p) {
    constexpr int KS = 256 / 16;                             // K steps of an item
    constexpr uint32_t W_CHUNK = PB * 32 * KC * 2, W_BYTES = 4 * W_CHUNK;     // resident weights, per 64-deep chunk / all
    constexpr uint32_t STG_PLANE = TILE_M * 32 * 2;          // staging: one output plane of an item
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t w_full, full_bar[2], empty_bar[2];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const XbConvGeom &g = p.g;
    const uint32_t win_stage = ((uint32_t)p.win_rows * p.win_slot + 1023u) & ~1023u;     // as fwd_win_setup
    const uint32_t stg_off = W_BYTES + 2u * win_stage, stg_buf = (uint32_t)p.p_out * STG_PLANE;
    const int64_t n_items = (p.M + TILE_M - 1) / TILE_M;
    if (tid == 0) {
        mbar_init(&w_full, 1);
        for (int s = 0; s < 2; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], CONS_WARPS);
        }
        mbar_fence_init();
    }
    __syncthreads();
    const uint32_t smem_base = smem_u32(smem);
    if (smem_base & 1023u) __trap();                         // the 128-byte swizzle pattern repeats every 1024 B
    uint32_t t_wait[5] = {0, 0, 0, 0, 0};                   // role timing, slots as in conv_tc_kernel
    if (p.timing && blockIdx.x < 160 && (tid == 0 || tid == CONS_WARPS * 32)) xb_k12_timing[blockIdx.x][tid == 0 ? 0 : 4] = clock64();
    auto timed_wait = [&](uint64_t *bar, uint32_t parity, int slot) {
        if (p.timing) {
            const uint32_t t0 = clock32();
            mbar_wait(bar, parity);
            t_wait[slot] += clock32() - t0;
        } else {
            mbar_wait(bar, parity);
        }
    };

    if (warp >= CONS_WARPS) {
        // ------------------------------------------------------------------ producer: one thread issues every copy
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
        if (tid == CONS_WARPS * 32) {
            mbar_expect_tx(&w_full, W_BYTES);
#pragma unroll
            for (int kc = 0; kc < 4; ++kc) tma_load_3d(smem_base + kc * W_CHUNK, &p.tm_b, kc * KC, 0, 0, &w_full);
            const uint32_t bytes = (uint32_t)(p.win_rows * p.win_kh * p.win_w * 16);
            uint32_t it = 0;
            for (int64_t w = blockIdx.x; w < n_items; w += gridDim.x, ++it) {
                const uint32_t stage = it & 1u;
                timed_wait(&empty_bar[stage], ((it >> 1) & 1u) ^ 1u, 0);
                const uint32_t base = smem_base + W_BYTES + stage * win_stage;
                const int64_t R0 = xb_div((uint32_t)(w * TILE_M), g.div_ox);      // first grid row of the item
                mbar_expect_tx(&full_bar[stage], bytes);
                for (int j = 0; j < p.win_rows; ++j) {
                    int b, iy0;
                    xb_win_box(g, R0 + j, b, iy0);
                    // 8-byte elements: unit u is elements 2u, 2u + 1
                    tma_load_3d(base + (uint32_t)j * p.win_slot, &p.tm_a, 2 * g.dx[0], iy0, b, &full_bar[stage]);
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ consumers: wgmma issue + epilogue
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONS_REGS));
        const int wg = warp >> 2;
        // this lane's ldmatrix row (see conv_tc_kernel): site m_l + lr of the warpgroup's 64, K unit 2 ks + (mi >> 1)
        const int mi = lane >> 3, lr = lane & 7, m_l = 16 * (warp & 3) + 8 * (mi & 1);
        uint32_t tap_off[KS];
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) tap_off[ks] = xb_win_tap_off(g, 8 * (2 * ks + (mi >> 1)), p.win_w);
        const int rbase = 64 * wg + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
        float bias[4][2];                                    // this thread's 8 columns 8 i + cq + e
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) bias[i][e] = p.bias ? p.bias[8 * i + cq + e] : 0.f;
        // B as in conv_tc_kernel's forward with b_tma: K step of 16 = 32 B within a chunk, chunks W_CHUNK apart
        const uint64_t b0 = make_desc_sw128(0, 16, 1024) + (uint64_t)(smem_base >> 4);
        timed_wait(&w_full, 0, 0);
        float acc[PB][16];
        uint32_t it = 0;
        for (int64_t w = blockIdx.x; w < n_items; w += gridDim.x, ++it) {
            const uint32_t stage = it & 1u;
            const int64_t m0 = w * TILE_M;
            const int64_t R0 = xb_div((uint32_t)m0, g.div_ox);      // first grid row of the item
            const uint32_t row = smem_base + W_BYTES + stage * win_stage + xb_win_site_off(g, m0 + 64 * wg + m_l + lr, R0, p.win_slot);
            timed_wait(&full_bar[stage], (it >> 1) & 1u, 0);
            // every fragment of the item is loaded while no wgmma is in flight (see conv_tc_kernel)
            uint32_t af[KS][4];
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) ldmatrix_x4<0>(af[ks], row + tap_off[ks]);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < KS; ++ks)
                mma_plane<0, PB, 1, 0>(acc, af[ks], b0 + (uint64_t)(((ks >> 2) * W_CHUNK + (ks & 3) * 32) >> 4), ks == 0 ? 0u : 1u);
            wgmma_commit();
            timed_wgmma_wait<0>(p.timing, t_wait[3]);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
            const uint32_t t_epi = p.timing ? clock32() : 0u;
            // ---- epilogue: rows rbase (h = 0) and rbase + 8 (h = 1) into the staging tile, groups added smallest first
            uint8_t *stg = smem + stg_off + stage * stg_buf;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float v[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        v[e] = acc[PB - 1][4 * i + 2 * h + e];
#pragma unroll
                        for (int gq = PB - 2; gq >= 0; --gq) v[e] += acc[gq][4 * i + 2 * h + e];
                        v[e] += bias[i][e];
                        if (p.relu) v[e] = fmaxf(v[e], 0.f);
                    }
                    __nv_bfloat16 q0[3], q1[3];
                    split3_bf16(v[0], q0[0], q0[1], q0[2]);
                    split3_bf16(v[1], q1[0], q1[1], q1[2]);
                    uint8_t *dst = stg + (rbase + 8 * h) * 64 + (8 * i + cq) * 2;
#pragma unroll
                    for (int q = 0; q < 3; ++q)
                        if (q < p.p_out) *reinterpret_cast<uint32_t *>(dst + q * STG_PLANE) = pack2(q0[q], q1[q]);
                }
            fence_proxy_async();           // written by the generic proxy, read by the bulk copies (async proxy)
            // the copies of the item before this one have read the other staging tile: free for the next item
            if (warp == 0) bulk_wait_read_all();
            asm volatile("bar.sync 1, %0;" ::"n"(CONS_WARPS * 32) : "memory");
            if (warp == 0 && lane < p.win_rows) {
                // lane j: the sites of grid row R0 + j in this item, consecutive pixels of one output row
                const int64_t R = R0 + lane, m1 = m0 + TILE_M < p.M ? m0 + TILE_M : p.M;
                const int64_t s0 = R * g.OX > m0 ? R * g.OX : m0, s1 = (R + 1) * g.OX < m1 ? (R + 1) * g.OX : m1;
                if (s0 < s1) {
                    int b, y, x;
                    xb_conv_site(g, s0, b, y, x);
                    const int64_t orow = (((int64_t)b * p.out_H + y * p.oys + p.oy0) * p.out_W + x + p.ox0) * 32;
                    const uint32_t src = smem_u32(stg) + (uint32_t)(s0 - m0) * 64u, n = (uint32_t)(s1 - s0) * 64u;
                    for (int q = 0; q < p.p_out; ++q) bulk_store(p.out[q] + orow, src + q * STG_PLANE, n);
                }
                bulk_commit();
            }
            if (p.timing) t_wait[4] += clock32() - t_epi;
        }
        if (warp == 0) bulk_wait_all();
    }
    if (p.timing && blockIdx.x < 160) {
        const unsigned long long now = clock64();
        unsigned long long *o = xb_k12_timing[blockIdx.x];
        if (tid == 0) o[0] = now - o[0], o[1] = t_wait[0], o[2] = t_wait[3], o[3] = 0, o[7] = t_wait[4];
        if (tid == CONS_WARPS * 32) o[4] = now - o[4], o[5] = t_wait[0], o[6] = 0;
    }
}

// The data gradient of a stride-2 layer as four stride phases (py, px) of N = 32 columns over a resident halo tile (three
// planes each side, bf16 plane outputs whose pixels are 64-byte rows, ReLU mask and column sums, no bias or fp32 output;
// selected by xb_gemm_halo_tc) - conv2's data gradient into g1.  Work items, mainloop and producer are conv_tc_kernel's in
// halo mode: an M tile of 128 positions with its four sub-items back to back on the same halo tile, the same n32 wgmmas
// on the same fragments, B planes and accumulators in the same order, groups added smallest first.  Only the epilogue
// differs, and not in its arithmetic:
//   * staging: phases (py, 0) and (py, 1) are consecutive sub-items and write every pixel of the output rows of the tile's
//     raster rows (conv_index.h, xb_pair_*).  The consumers write their split planes into a staging tile laid out as those
//     rows, [plane][slot = raster row - xb_pair_row0][out_W pixels][64 B], and after the second phase a helper thread of
//     the producer warpgroup stores each run of pixels with one cp.async.bulk per plane.  Nothing else of the output is
//     written (padding rows stay untouched).  The first phase of the next pair writes the tile once those stores have
//     read it (stg_empty);
//   * mask: each consumer loads its 8 mask words of a sub-item BEFORE the sub-item's MMAs, which hide their latency.  (The
//     masks bulk-copied into staging plane 0 measured slower: that load can start only when the previous pair's stores
//     have read the tile, and one sub-item of MMAs does not cover it; beside the tile there is no room for them.);
//   * column sums: the per-warp shuffle sums go to s_colsum[tile parity][sub-item][warp], and the tile's four column-sum
//     rows are added in the same fixed warp order after ONE consumer barrier per tile.
// The outputs and column sums are therefore bit for bit those of conv_tc_kernel<false, 3, 3, 1>.
__global__ void __launch_bounds__(THREADS, 1) conv_tc_kernel_dgrad_phases(const __grid_constant__ ConvParams p) {
    constexpr int PA = 3, PB = 3, NC = 1, N = 32, N_SUB = 4;
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t full_bar[MAX_STAGES], empty_bar[MAX_STAGES], a_full[2], a_empty[2], stg_full, stg_empty;
    __shared__ float s_colsum[2][N_SUB][CONS_WARPS][N];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int S = p.stages, n_chunks = p.halo_chunks, n_slots = xb_pair_slots(p.halo_w);
    const uint32_t w_plane = xb_conv_w_plane_bytes(N), stage_bytes = PB * w_plane;
    const uint32_t halo_plane = ((uint32_t)(p.halo_rows * p.halo_w) * 128u + 1023u) & ~1023u;
    const uint32_t a_buf_bytes = PA * halo_plane, ring_off = 2u * a_buf_bytes;
    // staging: p_out planes of n_slots output rows, as dgrad_phases_setup
    const uint32_t slot_bytes = (uint32_t)p.out_W * 64u, stg_plane = (uint32_t)n_slots * slot_bytes;
    const uint32_t stg_off = ring_off + (uint32_t)S * stage_bytes;
    const int64_t n_work = (p.halo_positions + TILE_M - 1) / TILE_M;
    const uint32_t raster_rows = (uint32_t)(p.halo_positions / p.halo_w);
    auto halo_row_lo = [&](int64_t t) -> int {              // as conv_tc_kernel
        const uint32_t num = (uint32_t)(t * TILE_M + p.halo_lo + 4 * p.halo_w);
        return (int)xb_div(num, p.halo_div_w) - 4;
    };
    // output row of raster row R in row phase py (-1: none)
    auto out_row = [&](uint32_t R, int py) -> int64_t {
        return xb_pair_out_row(R, raster_rows, p.box_div_hp, p.box_hp, p.box_y0, p.sub_y1[2 * py], p.sub_oy0[2 * py], p.out_H);
    };
    auto run_of = [&](int64_t p0, uint32_t R, int py, int &lo, int &hi) -> int {
        return xb_pair_run(p0, R, p.halo_w, p.halo_w0, p.sub_x1[2 * py], p.sub_x1[2 * py + 1], lo, hi);
    };

    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], CONS_WARPS);
        }
        for (int a = 0; a < 2; ++a) {
            mbar_init(&a_full[a], 1);
            mbar_init(&a_empty[a], CONS_WARPS);
        }
        mbar_init(&stg_full, CONS_WARPS);
        mbar_init(&stg_empty, 1);
        mbar_fence_init();
    }
    __syncthreads();
    const uint32_t smem_base = smem_u32(smem);
    if (smem_base & 1023u) __trap();                         // the 128-byte swizzle pattern repeats every 1024 B
    uint32_t t_wait[5] = {0, 0, 0, 0, 0};                   // role timing, slots as in conv_tc_kernel
    if (p.timing && blockIdx.x < 160 && (tid == 0 || tid == CONS_WARPS * 32)) xb_k12_timing[blockIdx.x][tid == 0 ? 0 : 4] = clock64();
    auto timed_wait = [&](uint64_t *bar, uint32_t parity, int slot) {
        if (p.timing) {
            const uint32_t t0 = clock32();
            mbar_wait(bar, parity);
            t_wait[slot] += clock32() - t0;
        } else {
            mbar_wait(bar, parity);
        }
    };

    if (warp >= CONS_WARPS) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
        if (tid == CONS_WARPS * 32) {
            // ---------------------------------------------------------------- producer: halo tiles and the weight ring
            uint32_t it = 0, tile_it = 0;
            for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x, ++tile_it) {
                const uint32_t buf = tile_it & 1u;
                timed_wait(&a_empty[buf], ((tile_it >> 1) & 1u) ^ 1u, 1);
                mbar_expect_tx(&a_full[buf], (uint32_t)PA * (uint32_t)(p.halo_rows * p.halo_w) * 128u);
                const int r_lo = halo_row_lo(w);
#pragma unroll
                for (int q = 0; q < PA; ++q)
                    tma_load_box(smem_base + buf * a_buf_bytes + q * halo_plane, &p.tm_a, 0, p.halo_w0, r_lo, 1, q, &a_full[buf]);
                for (int kc = 0; kc < N_SUB * n_chunks; ++kc, ++it) {
                    const int stage = (int)(it % (uint32_t)S);
                    timed_wait(&empty_bar[stage], ((it / (uint32_t)S) & 1u) ^ 1u, 0);
                    mbar_expect_tx(&full_bar[stage], stage_bytes);
                    tma_load_3d(smem_base + ring_off + (uint32_t)stage * stage_bytes, &p.tm_b, (kc % n_chunks) * KC,
                                (kc / n_chunks) * N, 0, &full_bar[stage]);
                }
            }
        } else if (tid == CONS_WARPS * 32 + 32) {
            // ---------------------------------------------------------------- staging: output runs out
            const uint32_t stg = smem_base + stg_off;
            uint32_t k = 0;                                  // phase pairs so far
            for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x) {
                const int64_t p0 = w * TILE_M;
                const uint32_t R0 = xb_pair_row0(p0, p.halo_div_w);
                for (int py = 0; py < 2; ++py, ++k) {
                    mbar_wait(&stg_full, k & 1u);            // the consumers have written both phases of the pair
                    for (int j = 0; j < n_slots; ++j) {
                        int lo, hi;
                        const int64_t orw = out_row(R0 + j, py);
                        if (orw >= 0 && run_of(p0, R0 + j, py, lo, hi) > 0)
                            for (int q = 0; q < p.p_out; ++q)
                                bulk_store(p.out[q] + (orw * p.out_W + lo) * 32, stg + q * stg_plane + j * slot_bytes + lo * 64,
                                           (uint32_t)(hi - lo + 1) * 64u);
                    }
                    bulk_commit();
                    bulk_wait_read_all();
                    mbar_arrive(&stg_empty);                 // the stores have read the staging tile: free for the next pair
                }
            }
            bulk_wait_all();
        }
    } else {
        // ------------------------------------------------------------------ consumers: wgmma issue + epilogue
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONS_REGS));
        const int wg = warp >> 2;
        const uint64_t b_tmpl = make_desc_sw128(0, 16, 1024);    // as conv_tc_kernel's forward with b_tma: K step of 16 = 32 B
        const int mi = lane >> 3, lr = lane & 7, m_l = 16 * (warp & 3) + 8 * (mi & 1);
        const uint32_t a_lane = (uint32_t)wg * 8192u + (uint32_t)(m_l + lr) * 128u;
        const int rbase = 64 * wg + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
        float acc[PB * NC][16];
        uint32_t it = 0, tile_it = 0, k = 0;
        for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x, ++tile_it) {
            const uint32_t buf = tile_it & 1u;
            timed_wait(&a_full[buf], (tile_it >> 1) & 1u, 2);
            const uint32_t halo_base = smem_base + buf * a_buf_bytes;
            const int halo_s0 = (int)(w * TILE_M) - halo_row_lo(w) * p.halo_w;     // tile row of the site of MMA row 0
            // this thread's two rows: raster pixel (x, y), their staging byte offset and their mask element at pixel 2x of
            // output row 2 (y - y0) of the image
            const int64_t p0 = w * TILE_M;
            const uint32_t R0 = xb_pair_row0(p0, p.halo_div_w);
            int rx[2], ry[2];
            bool row_ok[2];
            uint32_t srow[2];
            int64_t mrow[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t P = p0 + rbase + 8 * h;
                const uint32_t R = xb_div((uint32_t)P, p.halo_div_w), b = xb_div(R, p.box_div_hp);
                rx[h] = (int)((uint32_t)P - R * (uint32_t)p.halo_w) + p.halo_w0;
                ry[h] = (int)(R - b * (uint32_t)p.box_hp);
                row_ok[h] = P < p.halo_positions && rx[h] >= 0 && ry[h] >= p.box_y0;
                srow[h] = (R - R0) * slot_bytes + (uint32_t)(rx[h] > 0 ? rx[h] : 0) * 128u;
                mrow[h] = (((int64_t)b * p.out_H + 2 * (ry[h] - p.box_y0)) * p.mask_W + 2 * rx[h] + p.mask_x0) * 32;
            }
            for (int sub = 0; sub < N_SUB; ++sub) {
                const int px = sub & 1;
                bool live[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) live[h] = row_ok[h] && rx[h] <= p.sub_x1[sub] && ry[h] <= p.sub_y1[sub];
                // the ReLU mask of this thread's 16 elements, loaded before the sub-item's MMAs (which hide the latency)
                uint32_t mw[4][2];
                {
                    const int64_t m_off = ((int64_t)p.sub_oy0[sub] * p.mask_W + px) * 32 + cq;
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            mw[i][h] = live[h] ? *reinterpret_cast<const uint32_t *>(p.mask + mrow[h] + m_off + 8 * i) : 0u;
                }
                uint32_t scale_d = 0;
                uint32_t af[KC / 16][PA][4];
                for (int kc = 0; kc < n_chunks; ++kc, ++it) {
                    const int stage = (int)(it % (uint32_t)S);
                    timed_wait(&full_bar[stage], (it / (uint32_t)S) & 1u, 0);
                    const uint32_t w_addr = smem_base + ring_off + (uint32_t)stage * stage_bytes;
                    const uint32_t a_row = a_lane + halo_base + (uint32_t)(halo_s0 + p.halo_shift[sub * n_chunks + kc]) * 128u;
                    const uint32_t a_sw = (a_row >> 7) & 7u;
                    const uint64_t b0 = b_tmpl + (uint64_t)(w_addr >> 4);
#pragma unroll
                    for (int ks = 0; ks < KC / 16; ++ks) {
                        const uint32_t a_addr = a_row + (((uint32_t)(2 * ks + (mi >> 1))) ^ a_sw) * 16u;
#pragma unroll
                        for (int q = 0; q < PA; ++q) ldmatrix_x4<0>(af[ks][q], a_addr + (uint32_t)q * halo_plane);
                    }
                    wgmma_fence();
#pragma unroll
                    for (int ks = 0; ks < KC / 16; ++ks) {
                        const uint64_t db = b0 + (uint64_t)(ks * (32 >> 4));
                        mma_plane<0, PB, NC, 0>(acc, af[ks][0], db, scale_d);
                        mma_plane<0, PB, NC, 1>(acc, af[ks][1], db, 1u);
                        mma_plane<0, PB, NC, 2>(acc, af[ks][2], db, 1u);
                        scale_d = 1;
                    }
                    wgmma_commit();
                    timed_wgmma_wait<0>(p.timing, t_wait[3]);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[stage]);
                }
                const uint32_t t_epi = p.timing ? clock32() : 0u;
                // ---- epilogue: rows rbase (h = 0) and rbase + 8 (h = 1) into the staging tile
                if (px == 0) mbar_wait(&stg_empty, (k & 1u) ^ 1u);     // the previous pair's stores have read the tile
                uint8_t *dst[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) dst[h] = smem + stg_off + srow[h] + px * 64;
                // the mask as one bit per element (bf16 > 0 <=> sign bit clear and not (+)zero), as conv_tc_kernel keeps it
                uint32_t keep = 0u;
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint32_t lo16 = mw[i][h] & 0xffffu, hi16 = mw[i][h] >> 16;
                        keep |= (uint32_t)(lo16 != 0u && lo16 < 0x8000u) << (4 * (2 * i + h));
                        keep |= (uint32_t)(hi16 != 0u && hi16 < 0x8000u) << (4 * (2 * i + h) + 1);
                    }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int c = 8 * i + cq;                                  // columns c, c + 1
                    float cs[2] = {0.f, 0.f};
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float v[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            v[e] = acc[PB - 1][4 * i + 2 * h + e];             // smallest group first
#pragma unroll
                            for (int gq = PB - 2; gq >= 0; --gq) v[e] += acc[gq][4 * i + 2 * h + e];
                            v[e] += 0.f;                                       // conv_tc_kernel's zero bias: -0 -> +0
                            if (!((keep >> (4 * (2 * i + h) + e)) & 1u)) v[e] = 0.f;
                        }
                        if (live[h]) {
                            __nv_bfloat16 q0[3], q1[3];
                            split3_bf16(v[0], q0[0], q0[1], q0[2]);
                            split3_bf16(v[1], q1[0], q1[1], q1[2]);
#pragma unroll
                            for (int q = 0; q < 3; ++q)
                                if (q < p.p_out) *reinterpret_cast<uint32_t *>(dst[h] + q * stg_plane + c * 2) = pack2(q0[q], q1[q]);
                            cs[0] += v[0], cs[1] += v[1];
                        }
                    }
#pragma unroll
                    for (int off = 4; off <= 16; off <<= 1) {
                        cs[0] += __shfl_xor_sync(0xffffffffu, cs[0], off);
                        cs[1] += __shfl_xor_sync(0xffffffffu, cs[1], off);
                    }
                    if (lane < 4) s_colsum[buf][sub][warp][c] = cs[0], s_colsum[buf][sub][warp][c + 1] = cs[1];
                }
                if (px == 1) {
                    // both phases of the pair are staged: hand the tile to the stores
                    fence_proxy_async();   // written by the generic proxy, read by the bulk copies (async proxy)
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&stg_full);
                    ++k;
                }
                if (p.timing) t_wait[4] += clock32() - t_epi;
            }
            // every MMA of this tile has retired (wait above): the halo tile is free
            __syncwarp();
            if (lane == 0) mbar_arrive(&a_empty[buf]);
            const uint32_t t_epi = p.timing ? clock32() : 0u;
            // the tile's column-sum rows, warps added in a fixed order (deterministic) as conv_tc_kernel does
            asm volatile("bar.sync 1, %0;" ::"n"(CONS_WARPS * 32) : "memory");
            for (int i = tid; i < N_SUB * N; i += CONS_WARPS * 32) {
                const int sub = i / N, c = i - sub * N;
                float s = s_colsum[buf][sub][0][c];
#pragma unroll
                for (int q = 1; q < CONS_WARPS; ++q) s += s_colsum[buf][sub][q][c];
                p.colsum[(w * N_SUB + sub) * (int64_t)N + c] = s;
            }
            if (p.timing) t_wait[4] += clock32() - t_epi;
        }
    }
    if (p.timing && blockIdx.x < 160) {
        const unsigned long long now = clock64();
        unsigned long long *o = xb_k12_timing[blockIdx.x];
        if (tid == 0) o[0] = now - o[0], o[1] = t_wait[0], o[2] = t_wait[3], o[3] = t_wait[2], o[7] = t_wait[4];
        if (tid == CONS_WARPS * 32) o[4] = now - o[4], o[5] = t_wait[0], o[6] = t_wait[1];
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
               int64_t plane_stride, int box_rows, int box_cols = 64, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) return false;
    if (((uintptr_t)base & 15) || (row_stride * 2) % 16 || (plane_stride * 2) % 16 || box_rows > 256) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)planes};
    const cuuint64_t strides[2] = {(cuuint64_t)row_stride * 2, (cuuint64_t)(planes > 1 ? plane_stride : row_stride * rows) * 2};
    const cuuint32_t box[3] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows, (cuuint32_t)planes};
    const cuuint32_t estr[3] = {1, 1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(base), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// input windows of conv_tc_kernel_wgrad_win: the [B, IH, IW, 8] bf16 plane as [B][IH][2 IW] 8-byte elements (a box row of
// 16-byte units would exceed the 256-element box limit as bf16), boxes of {2 win_w elements, KH rows, one image}, no swizzle,
// zero fill outside the input
bool make_tmap_win(CUtensorMap *tm, const void *base, int B, int IH, int IW, int win_w, int KH) {
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc || ((uintptr_t)base & 15)) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)IW * 2, (cuuint64_t)IH, (cuuint64_t)B};
    const cuuint64_t strides[2] = {(cuuint64_t)IW * 16, (cuuint64_t)IH * IW * 16};
    const cuuint32_t box[3] = {(cuuint32_t)win_w * 2, (cuuint32_t)KH, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 3, const_cast<void *>(base), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// pixel-pair windows of conv_tc_kernel_wgrad_pairs: the [planes][B][IH][IW][32] bf16 input as {64 channels, IW / 2 pairs,
// IH rows, B images, planes}, boxes of {64 channels, win_w pairs, one row, one image, every plane}, 128-byte swizzle, zero
// fill outside the image (an image's last rows never read the next image's first ones)
bool make_tmap_pairs(CUtensorMap *tm, const void *base, int64_t plane_stride, int planes, int B, int IH, int IW, int win_w) {
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc || ((uintptr_t)base & 15) || (plane_stride * 2) % 16 || IW % 2 || win_w > 256) return false;
    const cuuint64_t row_b = (cuuint64_t)IW * 64, img_b = (cuuint64_t)IH * row_b;
    const cuuint64_t dims[5] = {64, (cuuint64_t)IW / 2, (cuuint64_t)IH, (cuuint64_t)B, (cuuint64_t)planes};
    const cuuint64_t strides[4] = {128, row_b, img_b, planes > 1 ? (cuuint64_t)plane_stride * 2 : img_b * B};
    const cuuint32_t box[5] = {64, (cuuint32_t)win_w, 1, 1, (cuuint32_t)planes};
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void *>(base), dims, strides, box, estr,
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

// The window fields of p (conv_index.h, xb_win_*) for runs of `sites` consecutive sites, if the A operand is one plane of
// 16-byte units (C = 8) read through a full KH x KW tap rectangle in row-major order.
bool win_fields(ConvParams &p, int planes_a, int sites) {
    const XbConvGeom &g = p.g;
    if (planes_a != 1 || g.C != 8) return false;
    int KW = 1;
    while (KW < g.T && g.dy[KW] == g.dy[0]) ++KW;
    if (g.T % KW != 0) return false;
    for (int t = 0; t < g.T; ++t)
        if (g.dy[t] != g.dy[0] + t / KW || g.dx[t] != g.dx[0] + t % KW) return false;
    const int KH = g.T / KW, win_w = xb_win_width(g);
    if (2 * win_w > 256 || KH > 256 || p.M + sites >= ((int64_t)1 << 31)) return false;    // box limits, 32-bit site indices
    p.win_kh = KH, p.win_w = win_w, p.win_rows = xb_win_rows(g, sites);
    p.win_slot = ((uint32_t)(KH * win_w * 16) + 127u) & ~127u;             // TMA destinations 128-byte aligned
    return true;
}

// conv_tc_kernel_fwd_win takes a forward whose A operand is as in win_fields with K = 256, N = n_tile = 32 and bf16 plane
// outputs only (no fp32 output, mask or column sums), each site a contiguous 64-byte row of every output plane (oxs = 1,
// out_ld = 32, out_c0 = 0) - conv1 over raw pixels into act1.  Fills the window fields and the shared-memory size of p.
bool fwd_win_setup(ConvParams &p, int planes_a, int planes_b, int N, int n_tile) {
    const XbConvGeom &g = p.g;
    if (N != 32 || n_tile != 32 || g.T * g.C != 256 || p.p_out == 0 || p.out_f32 || p.mask || p.colsum) return false;
    if (p.oxs != 1 || p.out_ld != 32 || p.out_c0 != 0) return false;
    if (!win_fields(p, planes_a, TILE_M) || p.win_rows > 32) return false;
    if (p.M + TILE_M + (int64_t)p.win_rows * g.OX >= ((int64_t)1 << 31)) return false;  // the window's last grid row
    // resident weights, two window stages (1024-byte aligned as the kernel lays them out), two staging tiles
    const uint32_t win_stage = ((uint32_t)p.win_rows * p.win_slot + 1023u) & ~1023u;
    const uint32_t bytes = (uint32_t)planes_b * 32u * 256u * 2u + 2u * win_stage + 2u * (uint32_t)p.p_out * TILE_M * 64u;
    if (bytes > (uint32_t)XB_K12_MAX_DYN_SMEM) return false;
    p.stages = 2;
    p.dyn_smem = bytes;
    return true;
}

template <int PB>
int launch_fwd_win(const ConvParams &p, void *stream) {
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(conv_tc_kernel_fwd_win<PB>, cudaFuncAttributeMaxDynamicSharedMemorySize, XB_K12_MAX_DYN_SMEM);
        attr = true;
    }
    const int64_t items = (p.M + TILE_M - 1) / TILE_M;
    const int grid = (int)(items < xb_sm_count() ? items : xb_sm_count());
    conv_tc_kernel_fwd_win<PB><<<grid, THREADS, p.dyn_smem, (cudaStream_t)stream>>>(p);
    return xb_launch_status();
}

// conv_tc_kernel_wgrad_win takes a weight gradient whose A operand is one plane of 16-byte units (C = 8) read through a full
// KH x KW tap rectangle in row-major order, with N = n_tile = 32 and 64 <= K <= 256 (two m64 row blocks per consumer
// warpgroup) - conv1 over raw pixels, 4 channels folded in pixel pairs.  Fills the window fields and the ring of p.
bool wgrad_win_setup(ConvParams &p, int planes_a, int planes_b, int N, int n_tile) {
    const XbConvGeom &g = p.g;
    if (N != 32 || n_tile != 32 || g.T % 8 != 0 || g.T * g.C > 2 * TILE_M || !win_fields(p, planes_a, KC)) return false;
    // stage: the output-gradient box (4096 B per plane) + the window slots, 1024-byte aligned (the 64-byte swizzle
    // pattern of the box repeats every 512 B of absolute address)
    const uint32_t stage_bytes = ((uint32_t)planes_b * 4096u + (uint32_t)p.win_rows * p.win_slot + 1023u) & ~1023u;
    int stages = (int)((uint32_t)XB_K12_MAX_DYN_SMEM / stage_bytes);
    if (stages < 2) return false;
    p.stages = stages > MAX_STAGES ? MAX_STAGES : stages;
    p.dyn_smem = (uint32_t)p.stages * stage_bytes;
    return true;
}

template <int PB>
int launch_win(const ConvParams &p, void *stream) {
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(conv_tc_kernel_wgrad_win<PB>, cudaFuncAttributeMaxDynamicSharedMemorySize, XB_K12_MAX_DYN_SMEM);
        attr = true;
    }
    const int grid = p.splits < xb_sm_count() ? p.splits : xb_sm_count();
    conv_tc_kernel_wgrad_win<PB><<<grid, THREADS, p.dyn_smem, (cudaStream_t)stream>>>(p);
    return xb_launch_status();
}

// conv_tc_kernel_wgrad_pairs takes a weight gradient with three planes on each side whose A operand is a 32-channel input
// read through a full KH x 4 tap rectangle in row-major order with an even column stride and first column (each 128-row
// K tile is one tap row: two 64-channel pixel pairs per site), with N = n_tile = 64 - conv2 of BoxNatureCNN over act1.
// Fills the window fields and the ring of p.
bool wgrad_pairs_setup(ConvParams &p, int planes_a, int planes_b, int N, int n_tile) {
    const XbConvGeom &g = p.g;
    if (planes_a != 3 || planes_b != 3 || g.C != 32 || N != 64 || n_tile != 64 || g.T % XB_PWIN_KW != 0) return false;
    if (g.sx % 2 != 0 || g.dx[0] % 2 != 0 || g.IW % 2 != 0) return false;
    for (int t = 0; t < g.T; ++t)
        if (g.dy[t] != g.dy[0] + t / XB_PWIN_KW || g.dx[t] != g.dx[0] + t % XB_PWIN_KW) return false;
    const int win_w = xb_pwin_width(g);
    if (win_w <= 0 || win_w > 256 || p.M + KC >= ((int64_t)1 << 31)) return false;      // box limit, 32-bit site indices
    p.win_kh = 1, p.win_w = win_w, p.win_rows = xb_win_rows(g);
    // every slot 1024-byte aligned: TMA's swizzle phase of a box is then the same whether it follows the address or the
    // box's own rows
    p.win_slot = ((uint32_t)(3 * win_w * 128) + 1023u) & ~1023u;
    const uint32_t stage_bytes = 3u * xb_conv_w_plane_bytes(64) + (uint32_t)p.win_rows * p.win_slot;
    int stages = (int)((uint32_t)XB_K12_MAX_DYN_SMEM / stage_bytes);
    if (stages < 2) return false;
    p.stages = stages > MAX_STAGES ? MAX_STAGES : stages;
    p.dyn_smem = (uint32_t)p.stages * stage_bytes;
    return true;
}

// XB_K12_DGRAD_PHASES=0 keeps every halo launch on conv_tc_kernel (the reference conv_tc_kernel_dgrad_phases must equal)
bool dgrad_phases_enabled() {
    static int on = -1;
    if (on < 0) {
        const char *e = getenv("XB_K12_DGRAD_PHASES");
        on = (e && e[0] == '0') ? 0 : 1;
    }
    return on == 1;
}

// conv_tc_kernel_dgrad_phases takes a halo launch with three planes on each side and four stride phases of N = 32 columns
// that write the same output columns (same_cols) at oys = oxs = 2, in the order (py, px) = (0, 0), (0, 1), (1, 0), (1, 1),
// where the two phases of a py share their output rows and together write one run of consecutive pixels per raster row
// (conv_index.h, xb_pair_*); its outputs are bf16 planes only whose pixels are 64-byte rows (out_ld = 32, out_c0 = 0), with
// a ReLU mask of the same pixel rows and column sums, and without bias or ReLU - conv2's data gradient of BoxNatureCNN.
// Fills the ring and the shared-memory size of p (halo tiles a_bytes, weight stages, staging tile).
bool dgrad_phases_setup(ConvParams &p, int planes_a, int planes_b, int n_sub, int N, int same_cols, uint32_t a_bytes) {
    if (planes_a != 3 || planes_b != 3 || n_sub != 4 || N != 32 || !same_cols || p.oys != 2 || p.oxs != 2) return false;
    if (p.p_out == 0 || p.out_f32 || p.bias || p.relu || !p.mask || !p.colsum || p.out_ld != 32 || p.out_c0 != 0) return false;
    for (int py = 0; py < 2; ++py) {
        const int e = 2 * py, o = e + 1;
        if (p.sub_oy0[e] != p.sub_oy0[o] || p.sub_y1[e] != p.sub_y1[o] || p.sub_ox0[e] != 0 || p.sub_ox0[o] != 1) return false;
        if (p.sub_x1[o] != p.sub_x1[e] && p.sub_x1[o] != p.sub_x1[e] - 1) return false;
    }
    const uint32_t stg = (uint32_t)p.p_out * (uint32_t)xb_pair_slots(p.halo_w) * (uint32_t)p.out_W * 64u;
    const uint32_t stage_bytes = 3u * xb_conv_w_plane_bytes(32);
    if (a_bytes + stg + 2u * stage_bytes > (uint32_t)XB_K12_MAX_DYN_SMEM) return false;
    const int stages = (int)(((uint32_t)XB_K12_MAX_DYN_SMEM - a_bytes - stg) / stage_bytes);
    p.stages = stages > MAX_STAGES ? MAX_STAGES : stages;
    p.dyn_smem = a_bytes + (uint32_t)p.stages * stage_bytes + stg;
    return true;
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
    if (tma_enabled() && fwd_win_setup(p, planes_a, planes_b, N, n_tile)) {
        // input windows and resident weights by TMA, outputs by bulk copies (conv_tc_kernel_fwd_win)
        if (!make_tmap_win(&p.tm_a, in, B, IH, IW, p.win_w, p.win_kh) ||
            !make_tmap(&p.tm_b, w, (int64_t)T * C, N, planes_b, (int64_t)T * C, w_plane, n_tile))
            return XB_EINVAL;
        if (planes_b == 1) return launch_fwd_win<1>(p, stream);
        if (planes_b == 2) return launch_fwd_win<2>(p, stream);
        return launch_fwd_win<3>(p, stream);
    }
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
    if (dgrad_phases_enabled() && dgrad_phases_setup(p, planes_a, planes_b, n_sub, N, same_cols, a_bytes)) {
        // the stride phases by pairs: masks in and output rows out by bulk copies (conv_tc_kernel_dgrad_phases)
        static bool attr = false;
        if (!attr) {
            cudaFuncSetAttribute(conv_tc_kernel_dgrad_phases, cudaFuncAttributeMaxDynamicSharedMemorySize, XB_K12_MAX_DYN_SMEM);
            attr = true;
        }
        const int grid = (int)(tiles < xb_sm_count() ? tiles : xb_sm_count());
        conv_tc_kernel_dgrad_phases<<<grid, THREADS, p.dyn_smem, (cudaStream_t)stream>>>(p);
        return xb_launch_status();
    }
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
    if (tma_enabled() && wgrad_win_setup(p, planes_a, planes_b, N, n_tile)) {
        // both operands by TMA, one work item per split (conv_tc_kernel_wgrad_win)
        if (!make_tmap_win(&p.tm_a, in, B, IH, IW, p.win_w, p.win_kh) ||
            !make_tmap(&p.tm_b, g, N, p.M, planes_b, g_ld, g_plane, KC, 32, CU_TENSOR_MAP_SWIZZLE_64B))
            return XB_EINVAL;
        if (planes_b == 1) return launch_win<1>(p, stream);
        if (planes_b == 2) return launch_win<2>(p, stream);
        return launch_win<3>(p, stream);
    }
    if (tma_enabled() && wgrad_pairs_setup(p, planes_a, planes_b, N, n_tile)) {
        // both operands by TMA, the gathered path's work items (split, K tile) (conv_tc_kernel_wgrad_pairs)
        if (!make_tmap_pairs(&p.tm_a, in, in_plane, planes_a, B, IH, IW, p.win_w) ||
            !make_tmap(&p.tm_b, g, N, p.M, planes_b, g_ld, g_plane, KC))
            return XB_EINVAL;
        static bool attr = false;
        if (!attr) {
            cudaFuncSetAttribute(conv_tc_kernel_wgrad_pairs, cudaFuncAttributeMaxDynamicSharedMemorySize, XB_K12_MAX_DYN_SMEM);
            attr = true;
        }
        const int64_t work = (int64_t)(T * C / TILE_M) * splits;
        const int grid = (int)(work < xb_sm_count() ? work : xb_sm_count());
        conv_tc_kernel_wgrad_pairs<<<grid, THREADS, p.dyn_smem, (cudaStream_t)stream>>>(p);
        return xb_launch_status();
    }
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

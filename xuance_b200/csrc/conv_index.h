// Index arithmetic of the gathered-operand tensor-core GEMM (conv_tc.cu), kept free of CUDA so that the SAME functions
// are compiled into the kernel and into the host-side layout test (tests/csrc/conv_index_test.cpp, run by
// tests/test_conv_index.py): the test stages operands with these functions into an emulated shared-memory image, reads
// them back the way the wgmma shared-memory descriptors do and compares with a direct
// convolution.
//
// The GEMM:  D[m, n] = sum_k A[m, k] * W[n, k]
//   m  <-> one site (b, y, x) of an output grid [B, OY, OX]
//   k  <-> (tap t, channel c), k = t*C + c, C a multiple of 8
//   A[m, (t, c)] = in[b, y*sy + dy[t], x*sx + dx[t], c]     (zero outside [0,IH) x [0,IW))    NHWC input
// which covers
//   * forward convolution:      dy[t] = kh - pad, dx[t] = kw - pad, (sy, sx) = stride              (cnn.py:45-50)
//   * a fully connected layer:  one tap, IH = IW = OY = OX = 1, C = in_features
//   * data gradient, stride 1:  the flipped taps dy[t] = pad - kh over the output-gradient tensor
//   * data gradient, stride s:  one such GEMM per phase (y mod s, x mod s) with that phase's taps, sy = sx = 1
// Operands travel as TWO bf16 tensors each (x = hi + lo, see tc_common.cuh::split_bf16).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define XB_HD __host__ __device__ __forceinline__
#else
#define XB_HD inline
#endif

#define XB_CONV_MAX_TAPS 64
#define XB_CONV_KC 64           // K elements per pipeline stage (8 core matrices, 128 B per operand row)
#define XB_CONV_TILE_M 128      // rows per CTA tile (two warpgroups of 64)

#define XB_CONV_MAX_UNITS 1024  // 16-byte K units per GEMM row the tap table holds: K = T * C <= 8192
#define XB_CONV_PRODUCERS 256   // producer threads per CTA (8 warps)

// division by a launch-time constant d >= 1 for 0 <= n < 2^31:  n / d == umulhi(n, mul) >> shift   (mul == 0: d == 1)
struct XbDiv {
    uint32_t mul, shift;
};
inline XbDiv xb_div_make(uint32_t d) {
    XbDiv v = {0u, 0u};
    if (d > 1) {
        uint32_t lg = 0;
        while ((1ull << lg) < d) ++lg;                       // ceil(log2 d)
        const uint32_t p = 31 + lg;
        v.mul = (uint32_t)(((1ull << p) + d - 1) / d);
        v.shift = p - 32;
    }
    return v;
}
XB_HD uint32_t xb_div(uint32_t n, const XbDiv &v) {
#if defined(__CUDA_ARCH__)
    return v.mul ? (__umulhi(n, v.mul) >> v.shift) : n;
#else
    return v.mul ? (uint32_t)(((uint64_t)n * v.mul) >> 32) >> v.shift : n;
#endif
}

struct XbConvGeom {
    int B, IH, IW, C;           // input tensor [B, IH, IW, C] (bf16 planes), C % 8 == 0
    int OY, OX;                 // output grid per image
    int sy, sx;                 // input step per output step
    int T;                      // taps; K = T * C, K % XB_CONV_KC == 0
    int N;                      // GEMM columns of one work item (the tile width), N % 32 == 0
    XbDiv div_img, div_ox;      // divisions by OY*OX and OX (xb_geom_finish)
    int8_t dy[XB_CONV_MAX_TAPS], dx[XB_CONV_MAX_TAPS];
};
inline void xb_geom_finish(XbConvGeom &g) {
    g.div_img = xb_div_make((uint32_t)(g.OY * g.OX));
    g.div_ox = xb_div_make((uint32_t)g.OX);
}

// byte offset of element (r, k) of a [rows x KP] bf16 operand in the K-major no-swizzle canonical layout
// (8-row x 16-byte core matrices; K-adjacent cores 128 B apart; 8-row groups KP/8*128 B apart)
XB_HD uint32_t xb_canon_off(int r, int k, int KP) {
    return (uint32_t)((r >> 3) * (KP >> 3) * 128 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2);
}

// byte offset of element (mn, k) of a [MN x KP] bf16 operand in the MN-major no-swizzle canonical layout: a core matrix
// is 8 k-rows of 16 bytes (8 consecutive mn elements); K-adjacent cores 128 B apart (descriptor LBO), 8-mn groups
// KP/8*128 B apart (descriptor SBO) - the transpose of xb_canon_off inside each core matrix, same core placement.
// (cute/atom/mma_traits_sm100.hpp, make_umma_desc<Major::MN>, LayoutType::INTERLEAVE: ((T,1,m),(8,k)):((1,T,SBO),(1T,LBO)))
XB_HD uint32_t xb_canon_off_mn(int mn, int k, int KP) {
    return (uint32_t)((mn >> 3) * (KP >> 3) * 128 + (k >> 3) * 128 + (k & 7) * 16 + (mn & 7) * 2);
}

// site m -> (b, y, x); m < 2^31
XB_HD void xb_conv_site(const XbConvGeom &g, int64_t m, int &b, int &y, int &x) {
    const int per_img = g.OY * g.OX;
    b = (int)xb_div((uint32_t)m, g.div_img);
    const int rem = (int)((uint32_t)m - (uint32_t)b * (uint32_t)per_img);
    y = (int)xb_div((uint32_t)rem, g.div_ox);
    x = rem - y * g.OX;
}

// packed weight [N, (kh, kw, c)] element i  <-  torch weight [N, C, KH, KW] element xb_pack_weight_src(i, ...)
XB_HD int64_t xb_pack_weight_src(int64_t i, int C, int KH, int KW) {
    const int64_t K = (int64_t)C * KH * KW;
    const int64_t n = i / K;
    int64_t r = i - n * K;
    const int c = (int)(r % C);
    r /= C;
    const int kw = (int)(r % KW), kh = (int)(r / KW);
    return ((n * C + c) * KH + kh) * KW + kw;
}

// sites per split of the weight-gradient reduction: a multiple of the chunk length; 0 if `splits` would leave one empty
XB_HD int64_t xb_wgrad_sites_per_split(int64_t M, int splits) {
    int64_t per = (M + splits - 1) / splits;
    per = (per + XB_CONV_KC - 1) / XB_CONV_KC * XB_CONV_KC;
    return ((int64_t)(splits - 1) * per >= M) ? 0 : per;
}

// ---------------------------------------------------------------------------------------------------------------------
// Staging: what ONE of the 256 producer threads copies for one K chunk.  emit_a / emit_w receive (byte offset of the
// 16-byte unit inside plane 0 of that operand in the stage, element offset of its 8 source values or -1 for a zero unit);
// the kernel turns each call into one cp.async per plane, the host test writes an emulated shared memory.
//
// Everything that does not depend on the row is tabulated once per launch (XbUnit per 16-byte K unit: tap offsets and the
// element offset relative to the site's un-shifted pixel) and everything that does not depend on the chunk once per tile
// (XbSite per row): a unit then costs two adds, two unsigned compares and a select.  (The first version recomputed
// tap = k / C and the site by integer division for every unit; with ONE producer warp per scheduler those dependent
// instruction chains, not the loads, set the pace whatever the byte count.)
//
// Mapping (row-coalesced): in the canonical no-swizzle layouts the shared-memory bank of a 16-byte unit depends only on
// (row & 7) [K-major] / (site & 7) [MN-major], so a warp instruction is conflict-free as soon as its 32 lanes hold each of
// the 8 residues four times, which leaves the other lane bits free to walk along MEMORY-contiguous units: lane ->
// (residue = lane & 7, unit = lane >> 3), i.e. 8 rows x 4 consecutive units = 8 x 64 contiguous bytes per instruction
// (whole 32-byte sectors; a thread-per-row mapping uses half of every sector it fetches).
// Thread pt in [0,256): team = pt >> 7 takes K units team*4 .. team*4+3 of the chunk (forward) / the sites with
// (site >> 3) & 1 == team (weight gradient); w = (pt >> 5) & 3, rs = pt & 7, uo = (pt >> 3) & 3.
// ---------------------------------------------------------------------------------------------------------------------
struct XbUnit {
    int32_t off;                // (dy * IW + dx) * C + c: element offset relative to pixel (y*sy, x*sx) channel 0
    int16_t dy, dx;
};
XB_HD XbUnit xb_unit(const XbConvGeom &g, int ku) {
    const int k0 = ku * 8, t = k0 / g.C, c = k0 - t * g.C;
    XbUnit e;
    e.dy = g.dy[t], e.dx = g.dx[t];
    e.off = ((int)e.dy * g.IW + (int)e.dx) * g.C + c;
    return e;
}

struct XbSite {
    int64_t base;               // element offset of pixel (y*sy, x*sx), channel 0, of image b
    int32_t iy0, ix0;           // y*sy, x*sx; a row outside the problem has iy0 far below zero (every unit reads as zero)
};
XB_HD XbSite xb_site(const XbConvGeom &g, int64_t m, int64_t M) {
    XbSite s;
    s.base = 0, s.iy0 = -(1 << 24), s.ix0 = 0;
    if (m < M) {
        int b, y, x;
        xb_conv_site(g, m, b, y, x);
        s.iy0 = y * g.sy, s.ix0 = x * g.sx;
        s.base = (((int64_t)b * g.IH + s.iy0) * g.IW + s.ix0) * g.C;
    }
    return s;
}
XB_HD int64_t xb_unit_src(const XbConvGeom &g, const XbSite &s, const XbUnit &e) {
    const int iy = s.iy0 + e.dy, ix = s.ix0 + e.dx;
    return ((unsigned)iy < (unsigned)g.IH && (unsigned)ix < (unsigned)g.IW) ? s.base + e.off : (int64_t)-1;
}

// rows a producer thread feeds in the forward mapping: 32*w + 8*gi + rs, gi < 4 (both teams own the same rows)
XB_HD int xb_fwd_row(int pt, int gi) { return 32 * ((pt >> 5) & 3) + 8 * gi + (pt & 7); }

// forward / data-gradient GEMM (K-major operands): the thread's 4 rows x 1 K unit of A, and its share of the weight tile
template <class EmitA, class EmitW>
XB_HD void xb_stage_fwd(const XbConvGeom &g, const XbUnit *tab, int pt, const XbSite *sites, int kc, EmitA &&emit_a,
                        EmitW &&emit_w) {
    const int K = g.T * g.C;
    const int team = pt >> 7, w = (pt >> 5) & 3, rs = pt & 7, uo = (pt >> 3) & 3;
    const int u = team * 4 + uo;
    const XbUnit e = tab[kc * (XB_CONV_KC / 8) + u];
    for (int gi = 0; gi < 4; ++gi)
        emit_a(xb_canon_off(32 * w + 8 * gi + rs, u * 8, XB_CONV_KC), xb_unit_src(g, sites[gi], e));
    for (int j = w; j < (g.N >> 3); j += 4) {               // 8-row groups of the weight tile, dealt to the warps
        const int n = j * 8 + rs;
        emit_w(xb_canon_off(n, u * 8, XB_CONV_KC), (int64_t)n * K + kc * XB_CONV_KC + u * 8);
    }
}

// weight-gradient GEMM (MN-major operands): the chunk holds 64 consecutive sites starting at chunk_site0 (sites >=
// site_end are zero); the thread owns site pp = 16*w + 8*team + rs and the column units 4*quad + uo, quad < 4, of the
// tile's 128 (t, c) columns; the second operand is the output gradient G[site*g_ld + g_c0 + n]
template <class EmitA, class EmitG>
XB_HD void xb_stage_wgrad(const XbConvGeom &g, const XbUnit *tab, int pt, int64_t mt, int64_t chunk_site0, int64_t site_end,
                          int64_t M, int64_t g_ld, int g_c0, EmitA &&emit_a, EmitG &&emit_g) {
    const int K = g.T * g.C;
    const int team = pt >> 7, w = (pt >> 5) & 3, rs = pt & 7, uo = (pt >> 3) & 3;
    const int pp = 16 * w + 8 * team + rs;
    const int64_t site = chunk_site0 + pp;
    const bool in_run = site < site_end;
    const XbSite s = xb_site(g, in_run ? site : M, M);
    for (int quad = 0; quad < 4; ++quad) {
        const int u = quad * 4 + uo;
        const int64_t ku = mt * (XB_CONV_TILE_M / 8) + u;
        emit_a(xb_canon_off_mn(u * 8, pp, XB_CONV_KC), ku * 8 < K ? xb_unit_src(g, s, tab[ku]) : (int64_t)-1);
    }
    for (int j = uo; j < (g.N >> 3); j += 4)
        emit_g(xb_canon_off_mn(j * 8, pp, XB_CONV_KC), in_run ? site * g_ld + g_c0 + j * 8 : (int64_t)-1);
}

// ---------------------------------------------------------------------------------------------------------------------
// Weight gradient from input WINDOWS (conv_tc.cu, conv_tc_kernel_wgrad_win): one A plane, C == 8 (one 16-byte unit per
// tap), the taps the full KH x KW rectangle in row-major order.  A chunk of 64 consecutive sites touches at most
// xb_win_rows grid rows R = b * OY + y (all images in one sequence), starting at R0 = chunk_site0 / OX; window slot j holds
// the KH input rows sy * y + dy[0] .. + KH - 1 of grid row R0 + j, units dx[0] .. dx[0] + win_w - 1 of each, as TMA wrote
// them (one box per slot, zero outside the input and for grid rows past the last image).  Row (site s, k unit t) of the
// MN-major A operand is then the 16 bytes at  xb_win_site_off(s) + xb_win_tap_off(t)  of the window: the consumers read
// their ldmatrix rows from there, where the gathered path stages them with xb_stage_wgrad.
// ---------------------------------------------------------------------------------------------------------------------
// units per window row: every tap of every site of a grid row
XB_HD int xb_win_width(const XbConvGeom &g) { return g.sx * (g.OX - 1) + (g.dx[g.T - 1] - g.dx[0]) + 1; }
// grid rows a run of `sites` consecutive sites can touch (a weight-gradient chunk: XB_CONV_KC; a forward item: XB_CONV_TILE_M)
XB_HD int xb_win_rows(const XbConvGeom &g, int sites = XB_CONV_KC) { return (sites - 2 + g.OX) / g.OX + 1; }
// first input row and image of window slot R (grid row R; b >= B past the last image)
XB_HD void xb_win_box(const XbConvGeom &g, int64_t R, int &b, int &iy0) {
    int y, x;
    xb_conv_site(g, R * g.OX, b, y, x);
    iy0 = y * g.sy + g.dy[0];
}
// byte offset of tap unit kcol / 8 within a window slot (rows kcol >= K, which no output keeps, read tap 0)
XB_HD uint32_t xb_win_tap_off(const XbConvGeom &g, int kcol, int win_w) {
    const int t = kcol < g.T * g.C ? kcol / g.C : 0;
    return (uint32_t)(((g.dy[t] - g.dy[0]) * win_w + (g.dx[t] - g.dx[0])) * 16);
}
// byte offset of site s's slot and first unit within the window of the chunk whose first grid row is R0
XB_HD uint32_t xb_win_site_off(const XbConvGeom &g, int64_t s, int64_t R0, uint32_t slot_bytes) {
    int b, y, x;
    xb_conv_site(g, s, b, y, x);
    return (uint32_t)((int64_t)b * g.OY + y - R0) * slot_bytes + (uint32_t)(x * g.sx * 16);
}

// ---------------------------------------------------------------------------------------------------------------------
// Weight gradient from PIXEL-PAIR windows (conv_tc.cu, conv_tc_kernel_wgrad_pairs): C == 32 input channels read as
// 64-channel pixel pairs (128 bytes), the taps the full KH x 4 rectangle in row-major order, sx and dx[0] even.  A 128-row
// K tile mt is then tap row mt: rows (kw, c), kw = 0, 1 in pair x * sx / 2 + dx[0] / 2 and kw = 2, 3 in the next pair.
// Window slot j of a chunk holds input row sy * y + dy[KW * mt] of grid row R0 + j (all images in one sequence), pairs
// dx[0] / 2 .. + xb_pwin_width - 1, every plane: [plane][pair][128 B] with TMA's 128-byte swizzle, one box per slot from a
// tensor map with one dimension per image (zero fill for the rows an image does not have and past the last image).
// The 16 bytes of row (site s, K rows kcol .. kcol + 7) of plane q of the MN-major A operand are at
//   xb_sw128(window + xb_pwin_site_off(s) + xb_pwin_tap_off(kcol) + q * xb_pwin_width * 128)
// where the gathered path stages them with xb_stage_wgrad.
// ---------------------------------------------------------------------------------------------------------------------
#define XB_PWIN_KW 4            // taps per tap row: 4 x 32 channels = one 128-row K tile
// pairs per window row: every tap of every site of a grid row
XB_HD int xb_pwin_width(const XbConvGeom &g) { return (g.sx * (g.OX - 1) + g.dx[XB_PWIN_KW - 1] - g.dx[0]) / 2 + 1; }
// input row of window slot R (grid row R) for K tile mt, and its image (b >= B past the last image)
XB_HD void xb_pwin_box(const XbConvGeom &g, int64_t R, int mt, int &b, int &iy) {
    int y, x;
    xb_conv_site(g, R * g.OX, b, y, x);
    iy = y * g.sy + g.dy[XB_PWIN_KW * mt];
}
// byte offset of K rows kcol .. kcol + 7 (one tap, 8 channels) within a pair row, pairs counted from the site's first
// (kcol within the 128-row tile: taps 0, 1 in the first pair, 2, 3 in the second)
XB_HD uint32_t xb_pwin_tap_off(const XbConvGeom &g, int kcol) {
    const int kw = kcol / g.C, d = g.dx[kw] - g.dx[0];
    return (uint32_t)((d >> 1) * 128 + ((d & 1) * g.C + kcol % g.C) * 2);
}
// byte offset of site s's slot and pair within the window of the chunk whose first grid row is R0
XB_HD uint32_t xb_pwin_site_off(const XbConvGeom &g, int64_t s, int64_t R0, uint32_t slot_bytes) {
    int b, y, x;
    xb_conv_site(g, s, b, y, x);
    return (uint32_t)((int64_t)b * g.OY + y - R0) * slot_bytes + (uint32_t)(x * (g.sx / 2) * 128);
}
// the 128-byte swizzle as TMA applies it: the 16-byte unit (bits 4-6) XOR bits 7-9 of the shared-memory address
XB_HD uint32_t xb_sw128(uint32_t a) { return a ^ (((a >> 7) & 7u) << 4); }

// ---------------------------------------------------------------------------------------------------------------------
// Data gradient of a stride-2 layer by stride-phase PAIRS (conv_tc.cu, conv_tc_kernel_dgrad_phases): the halo raster's
// positions P = R * halo_w + hc (raster row R = b * hp + y, pixel x = hc + halo_w0) of the M tile whose first position is
// p0 are computed in the four phases (py, px) as sub-items; phase (py, px) writes output pixel 2x + px of output row
// xb_pair_out_row(R, py).  The phases (py, 0) and (py, 1) together write, for each raster row of the tile, ONE run of
// consecutive pixels of that output row (x1_odd is x1_even or x1_even - 1): the kernel stages the pair's outputs as whole
// output rows (slot R - xb_pair_row0 of the tile) and stores every run with one bulk copy per plane.  A raster row cut by a
// tile boundary gives two runs, each stored by its own tile.
// ---------------------------------------------------------------------------------------------------------------------
// raster rows an M tile can touch (staging slots)
XB_HD int xb_pair_slots(int halo_w) { return (XB_CONV_TILE_M - 2 + halo_w) / halo_w + 1; }
// first raster row of the M tile whose first position is p0 (slot 0)
XB_HD uint32_t xb_pair_row0(int64_t p0, const XbDiv &div_w) { return xb_div((uint32_t)p0, div_w); }
// output row of raster row R in the phases of row phase py (first output row oy0, valid raster rows y0 .. y1 of each image
// of hp rows, `rows` = B * hp raster rows); -1 if that pair writes no pixel of it
XB_HD int64_t xb_pair_out_row(uint32_t R, uint32_t rows, const XbDiv &div_hp, int hp, int y0, int y1, int oy0, int out_H) {
    if (R >= rows) return -1;
    const uint32_t b = xb_div(R, div_hp);
    const int y = (int)(R - b * (uint32_t)hp);
    if (y < y0 || y > y1) return -1;
    return (int64_t)b * out_H + 2 * (y - y0) + oy0;
}
// the run [lo, hi] of output pixels that the tile from p0 writes in raster row R: pixels 2x of the positions with
// 0 <= x <= x1_even and 2x + 1 of those with x <= x1_odd; returns hi - lo + 1 (0: no pixel)
XB_HD int xb_pair_run(int64_t p0, uint32_t R, int halo_w, int halo_w0, int x1_even, int x1_odd, int &lo, int &hi) {
    const int64_t r0 = (int64_t)R * halo_w;
    const int h0 = p0 > r0 ? (int)(p0 - r0) : 0;
    const int h1 = p0 + XB_CONV_TILE_M - 1 < r0 + halo_w - 1 ? (int)(p0 + XB_CONV_TILE_M - 1 - r0) : halo_w - 1;
    const int xa = h0 + halo_w0 > 0 ? h0 + halo_w0 : 0, xb = h1 + halo_w0;
    const int xe = xb < x1_even ? xb : x1_even, xo = xb < x1_odd ? xb : x1_odd;        // last x of each phase
    lo = xa <= xe ? 2 * xa : 2 * xa + 1;
    hi = 2 * xe > 2 * xo + 1 ? 2 * xe : 2 * xo + 1;
    if (xa > xe && xa > xo) lo = 0, hi = -1;
    return hi - lo + 1;
}

// shared-memory bytes of one pipeline stage: the P planes of A (hi | [mid |] lo) followed by the P planes of W.
// P = 2: x = hi + lo (|err| <= 2^-16 |x|, 3 products);  P = 3: x = hi + mid + lo (<= 2^-24 |x|, 6 products)
XB_HD uint32_t xb_conv_stage_bytes(int N, int P = 2) {
    return (uint32_t)(P * XB_CONV_TILE_M * XB_CONV_KC * 2 + P * N * XB_CONV_KC * 2);
}
XB_HD uint32_t xb_conv_a_plane_bytes() { return (uint32_t)(XB_CONV_TILE_M * XB_CONV_KC * 2); }
XB_HD uint32_t xb_conv_w_plane_bytes(int N) { return (uint32_t)(N * XB_CONV_KC * 2); }

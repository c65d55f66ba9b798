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

// shared-memory bytes of one pipeline stage: the P planes of A (hi | [mid |] lo) followed by the P planes of W.
// P = 2: x = hi + lo (|err| <= 2^-16 |x|, 3 products);  P = 3: x = hi + mid + lo (<= 2^-24 |x|, 6 products)
XB_HD uint32_t xb_conv_stage_bytes(int N, int P = 2) {
    return (uint32_t)(P * XB_CONV_TILE_M * XB_CONV_KC * 2 + P * N * XB_CONV_KC * 2);
}
XB_HD uint32_t xb_conv_a_plane_bytes() { return (uint32_t)(XB_CONV_TILE_M * XB_CONV_KC * 2); }
XB_HD uint32_t xb_conv_w_plane_bytes(int N) { return (uint32_t)(N * XB_CONV_KC * 2); }

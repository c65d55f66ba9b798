// Host emulation of conv_tc.cu's data movement, built by tests/test_conv_index.py with g++ (no CUDA needed).
// Staging uses the kernel's own index functions (xuance_b200/csrc/conv_index.h); the "tensor core" side re-derives the
// operand addresses from the shared-memory descriptor semantics that K9-TC validated on hardware (start address + ks*256,
// LBO = 128 B between K-adjacent core matrices, SBO = KC/8*128 B between 8-row groups, 16 B per core-matrix row), so a
// wrong placement by the producer shows up as a numeric mismatch (or a NaN from the poisoned stage).
#include <cmath>
#include <cstdint>
#include <limits>
#include <vector>

#include "../../xuance_b200/csrc/conv_index.h"

namespace {
inline float &at(std::vector<float> &smem, uint32_t byte_off) { return smem[byte_off / 2]; }   // one slot per bf16
}

// PA / PB planes of the A / B operand; N_total output columns in tiles of N (conv_tc.cu: work item = (m tile, n tile))
extern "C" int emul_gemm_gather(int PA, int PB, const float *in, int64_t in_plane, const float *w, int64_t w_plane, int B,
                                int IH, int IW, int C, int OY, int OX, int sy, int sx, int T, const int8_t *dy,
                                const int8_t *dx, int N_total, int N, int out_H, int out_W, int oys, int oxs, int oy0, int ox0,
                                int64_t out_ld, int out_c0, int stages, double *out) {
    if (PA < 1 || PA > PB || PB > 3 || N_total % N || PB * N > 256) return -2;
    XbConvGeom g;
    g.B = B, g.IH = IH, g.IW = IW, g.C = C, g.OY = OY, g.OX = OX, g.sy = sy, g.sx = sx, g.T = T, g.N = N;
    for (int t = 0; t < XB_CONV_MAX_TAPS; ++t) g.dy[t] = t < T ? dy[t] : 0, g.dx[t] = t < T ? dx[t] : 0;
    xb_geom_finish(g);
    const int KC = XB_CONV_KC, TM = XB_CONV_TILE_M, K = T * C;
    if (K % KC || C % 8 || N % 8 || K > 8 * XB_CONV_MAX_UNITS) return -1;
    std::vector<XbUnit> tab(K / 8);
    for (int i = 0; i < K / 8; ++i) tab[i] = xb_unit(g, i);
    const int n_chunks = K / KC;
    const uint32_t a_plane = xb_conv_a_plane_bytes(), ws_plane = xb_conv_w_plane_bytes(N);
    const uint32_t stage_bytes = PA * a_plane + PB * ws_plane;
    std::vector<float> smem((size_t)stages * stage_bytes / 2);
    const int64_t M = (int64_t)B * OY * OX, m_tiles = (M + TM - 1) / TM;
    const int n_tiles = N_total / N;
    const float nan = std::numeric_limits<float>::quiet_NaN();
    uint32_t it = 0;
    std::vector<double> acc((size_t)TM * PB * N);       // PB accumulator groups of N columns (accumulator columns g*N + n)
    for (int64_t work = 0; work < m_tiles * n_tiles; ++work) {
        const int64_t tile = work / n_tiles;
        const int nt = (int)(work % n_tiles);
        const int64_t w_off = (int64_t)nt * N * K;
        std::fill(acc.begin(), acc.end(), nan);         // accumulators start undefined: the first MMA must initialise every group
        for (int kc = 0; kc < n_chunks; ++kc, ++it) {
            const uint32_t base = (it % stages) * stage_bytes;
            for (uint32_t i = 0; i < stage_bytes / 2; ++i) smem[base / 2 + i] = nan;     // poison the stage
            // ---- producers (conv_tc.cu, warps 5-12): 256 threads, the staging routine and the tap table are the kernel's own
            for (int pt = 0; pt < XB_CONV_PRODUCERS; ++pt) {
                XbSite sites[4];
                for (int gi = 0; gi < 4; ++gi) sites[gi] = xb_site(g, tile * TM + xb_fwd_row(pt, gi), M);
                auto emit_a = [&](uint32_t dst, int64_t src) {
                    for (int q = 0; q < PA; ++q)
                        for (int j = 0; j < 8; ++j)
                            at(smem, base + q * a_plane + dst + 2 * j) = src >= 0 ? in[q * in_plane + src + j] : 0.f;
                };
                auto emit_w = [&](uint32_t dst, int64_t src) {
                    for (int q = 0; q < PB; ++q)
                        for (int j = 0; j < 8; ++j)
                            at(smem, base + PA * a_plane + q * ws_plane + dst + 2 * j) = src >= 0 ? w[q * w_plane + w_off + src + j] : 0.f;
                };
                xb_stage_fwd(g, tab.data(), pt, sites, kc, emit_a, emit_w);
            }
            // ---- tensor core (conv_tc.cu MMA warp): per K step of 16 ONE instruction per A plane pa, whose B operand is the
            // first (PB - pa) weight planes read as ONE matrix of (PB - pa) * N rows starting at the first plane (the planes
            // are adjacent in the stage, 8-row groups SBO apart), and whose result lands in accumulator columns
            // pa*N .. PB*N - 1; the very first instruction of a work item overwrites (accumulate = 0), all others add.
            const uint32_t LBO = 128, SBO = (KC / 8) * 128;
            const uint32_t w_addr = base + PA * a_plane;
            for (int ks = 0; ks < KC / 16; ++ks)
                for (int pa = 0; pa < PA; ++pa) {
                    const bool overwrite = (kc == 0 && ks == 0 && pa == 0);
                    const uint32_t sa = base + pa * a_plane + ks * 256, sb = w_addr + ks * 256;
                    const int NB = (PB - pa) * N;
                    for (int r = 0; r < TM; ++r)
                        for (int n = 0; n < NB; ++n) {
                            double s = 0.0;
                            for (int kk = 0; kk < 16; ++kk) {
                                const uint32_t inner = (kk >> 3) * LBO + (kk & 7) * 2;
                                const float av = at(smem, sa + (r >> 3) * SBO + (r & 7) * 16 + inner);
                                const float bv = at(smem, sb + (n >> 3) * SBO + (n & 7) * 16 + inner);
                                s += (double)av * (double)bv;
                            }
                            double &d = acc[(size_t)r * PB * N + pa * N + n];
                            d = overwrite ? s : d + s;
                        }
                }
        }
        // ---- epilogue: thread = row; the PB groups are added smallest first
        for (int r = 0; r < TM; ++r) {
            const int64_t m = tile * TM + r;
            if (m >= M) continue;
            int b, y, x;
            xb_conv_site(g, m, b, y, x);
            const int64_t orow = (((int64_t)b * out_H + (y * oys + oy0)) * out_W + (x * oxs + ox0)) * out_ld + out_c0 + (int64_t)nt * N;
            for (int n = 0; n < N; ++n) {
                double v = acc[(size_t)r * PB * N + (PB - 1) * N + n];
                for (int gq = PB - 2; gq >= 0; --gq) v += acc[(size_t)r * PB * N + gq * N + n];
                out[orow + n] = v;
            }
        }
    }
    return 0;
}

extern "C" void emul_pack_weight(const float *w, int N, int C, int KH, int KW, float *packed) {
    const int64_t total = (int64_t)N * C * KH * KW;
    for (int64_t i = 0; i < total; ++i) packed[i] = w[xb_pack_weight_src(i, C, KH, KW)];
}

// weight gradient (conv_tc_kernel<true>): partials[split, (t,c), n]; MN-major operands: the "tensor core" locates element
// (mn, k) at start + (mn/8)*SBO + (k/8)*LBO + (k%8)*16 + (mn%8)*2
extern "C" int emul_wgrad(int PA, int PB, const float *in, int64_t in_plane, const float *gr, int64_t g_plane, int64_t g_ld,
                          int B, int IH, int IW, int C, int OY, int OX, int sy, int sx, int T, const int8_t *dy,
                          const int8_t *dx, int N_total, int N, int splits, int stages, double *partials) {
    if (PA < 1 || PA > PB || PB > 3 || N_total % N || PB * N > 256) return -2;
    XbConvGeom g;
    g.B = B, g.IH = IH, g.IW = IW, g.C = C, g.OY = OY, g.OX = OX, g.sy = sy, g.sx = sx, g.T = T, g.N = N;
    for (int t = 0; t < XB_CONV_MAX_TAPS; ++t) g.dy[t] = t < T ? dy[t] : 0, g.dx[t] = t < T ? dx[t] : 0;
    xb_geom_finish(g);
    const int KC = XB_CONV_KC, TM = XB_CONV_TILE_M, K = T * C;
    if (K > 8 * XB_CONV_MAX_UNITS) return -1;
    std::vector<XbUnit> tab(K / 8);
    for (int i = 0; i < K / 8; ++i) tab[i] = xb_unit(g, i);
    const int64_t M = (int64_t)B * OY * OX;
    const int64_t per = xb_wgrad_sites_per_split(M, splits);
    if (per == 0 || C % 8 || N % 8) return -1;
    const uint32_t a_plane = xb_conv_a_plane_bytes(), ws_plane = xb_conv_w_plane_bytes(N);
    const uint32_t stage_bytes = PA * a_plane + PB * ws_plane;
    std::vector<float> smem((size_t)stages * stage_bytes / 2);
    const float nan = std::numeric_limits<float>::quiet_NaN();
    const int64_t m_tiles = (K + TM - 1) / TM;
    const int n_tiles = N_total / N;
    const int64_t mn_tiles = m_tiles * n_tiles;
    std::vector<double> acc((size_t)TM * PB * N);
    uint32_t it = 0;
    for (int64_t w = 0; w < mn_tiles * splits; ++w) {
        const int64_t sp = w / mn_tiles, rem = w - sp * mn_tiles;
        const int64_t mt = rem / n_tiles;
        const int nt = (int)(rem % n_tiles);
        const int64_t s0 = sp * per, site_end = (s0 + per < M) ? s0 + per : M;
        const int n_chunks = (int)((site_end - s0 + KC - 1) / KC);
        std::fill(acc.begin(), acc.end(), nan);
        for (int kc = 0; kc < n_chunks; ++kc, ++it) {
            const uint32_t base = (it % stages) * stage_bytes;
            for (uint32_t i = 0; i < stage_bytes / 2; ++i) smem[base / 2 + i] = nan;
            for (int pt = 0; pt < XB_CONV_PRODUCERS; ++pt) {
                auto emit_a = [&](uint32_t dst, int64_t src) {
                    for (int q = 0; q < PA; ++q)
                        for (int j = 0; j < 8; ++j)
                            at(smem, base + q * a_plane + dst + 2 * j) = src >= 0 ? in[q * in_plane + src + j] : 0.f;
                };
                auto emit_g = [&](uint32_t dst, int64_t src) {
                    for (int q = 0; q < PB; ++q)
                        for (int j = 0; j < 8; ++j)
                            at(smem, base + PA * a_plane + q * ws_plane + dst + 2 * j) = src >= 0 ? gr[q * g_plane + src + j] : 0.f;
                };
                xb_stage_wgrad(g, tab.data(), pt, mt, s0 + (int64_t)kc * KC, site_end, M, g_ld, nt * N, emit_a, emit_g);
            }
            const uint32_t LBO = 128, SBO = (KC / 8) * 128;
            const uint32_t w_addr = base + PA * a_plane;
            for (int ks = 0; ks < KC / 16; ++ks)
                for (int pa = 0; pa < PA; ++pa) {
                    const bool overwrite = (kc == 0 && ks == 0 && pa == 0);
                    const uint32_t sa = base + pa * a_plane + ks * 256, sb = w_addr + ks * 256;
                    const int NB = (PB - pa) * N;
                    for (int r = 0; r < TM; ++r)
                        for (int n = 0; n < NB; ++n) {
                            double s = 0.0;
                            for (int kk = 0; kk < 16; ++kk) {
                                const uint32_t inner = (kk >> 3) * LBO + (kk & 7) * 16;
                                const float av = at(smem, sa + (r >> 3) * SBO + inner + (r & 7) * 2);
                                const float bv = at(smem, sb + (n >> 3) * SBO + inner + (n & 7) * 2);
                                s += (double)av * (double)bv;
                            }
                            double &d = acc[(size_t)r * PB * N + pa * N + n];
                            d = overwrite ? s : d + s;
                        }
                }
        }
        for (int r = 0; r < TM; ++r) {
            const int64_t kcol = mt * TM + r;
            if (kcol >= K) continue;
            for (int n = 0; n < N; ++n) {
                double v = acc[(size_t)r * PB * N + (PB - 1) * N + n];
                for (int gq = PB - 2; gq >= 0; --gq) v += acc[(size_t)r * PB * N + gq * N + n];
                partials[((int64_t)sp * K + kcol) * N_total + (int64_t)nt * N + n] = v;
            }
        }
    }
    return 0;
}

// xb_wgrad_reduce: packed-layout partial sums -> torch [N, C, KH, KW]
extern "C" void emul_wgrad_reduce(const double *partials, int splits, int N, int C, int KH, int KW, double scale, double *dw) {
    const int64_t K = (int64_t)C * KH * KW, total = (int64_t)N * K;
    for (int64_t i = 0; i < total; ++i) {
        const int64_t n = i / K, k = i - n * K;
        double s = 0.0;
        for (int sp = 0; sp < splits; ++sp) s += partials[((int64_t)sp * K + k) * N + n];
        dw[xb_pack_weight_src(i, C, KH, KW)] = s * scale;
    }
}

// xb_div (multiply-high division by a launch-time constant): mismatches against n / d over [lo, hi) plus the top of the range
extern "C" int64_t emul_div_check(uint32_t d, uint32_t lo, uint32_t hi) {
    const XbDiv v = xb_div_make(d);
    int64_t bad = 0;
    for (uint32_t n = lo; n < hi; ++n) bad += xb_div(n, v) != n / d;
    for (uint32_t n = 0x7fffffffu - 4096; n <= 0x7fffffffu - 1; ++n) bad += xb_div(n, v) != n / d;
    return bad;
}

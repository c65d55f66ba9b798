// Host emulation of conv_tc_kernel_wgrad_win's A operand (conv_tc.cu), built by tests/test_conv_index_win.py with g++ (no
// CUDA needed); the index functions are the kernel's own (xuance_b200/csrc/conv_index.h).
#include <cstdint>
#include <limits>
#include <vector>

#include "../../xuance_b200/csrc/conv_index.h"

namespace {
inline float &at(std::vector<float> &smem, uint32_t byte_off) { return smem[byte_off / 2]; }   // one slot per bf16
}

// conv_tc_kernel_wgrad_win's A operand against the gathered path's: for every chunk of every split, the gathered stage of
// both 128-row tiles is built with xb_stage_wgrad and the input window as the TMA boxes of xb_win_box fill it (zero outside
// the input and past the last image); then every ldmatrix row address of every consumer lane, K step and row block is
// formed both ways (conv_tc.cu: the cp.async MN-major lane offset + ks * 256 in tile r, and xb_win_site_off + xb_win_tap_off)
// and the 8 values read there compared.  One plane, K = 2 * 128.  Returns the number of mismatching rows, -1 on bad input.
extern "C" int64_t emul_wgrad_win_check(const float *in, int B, int IH, int IW, int C, int OY, int OX, int sy, int sx, int T,
                                        const int8_t *dy, const int8_t *dx, int splits) {
    XbConvGeom g;
    g.B = B, g.IH = IH, g.IW = IW, g.C = C, g.OY = OY, g.OX = OX, g.sy = sy, g.sx = sx, g.T = T, g.N = 32;
    for (int t = 0; t < XB_CONV_MAX_TAPS; ++t) g.dy[t] = t < T ? dy[t] : 0, g.dx[t] = t < T ? dx[t] : 0;
    xb_geom_finish(g);
    const int KC = XB_CONV_KC, K = T * C;
    if (C != 8 || K != 2 * XB_CONV_TILE_M) return -1;
    std::vector<XbUnit> tab(K / 8);
    for (int i = 0; i < K / 8; ++i) tab[i] = xb_unit(g, i);
    const int64_t M = (int64_t)B * OY * OX, per = xb_wgrad_sites_per_split(M, splits);
    if (per == 0) return -1;
    int KW = 1;
    while (KW < T && g.dy[KW] == g.dy[0]) ++KW;
    const int KH = T / KW, win_w = xb_win_width(g), rows = xb_win_rows(g);
    const uint32_t slot = ((uint32_t)(KH * win_w * 16) + 127u) & ~127u, a_plane = xb_conv_a_plane_bytes();
    const float nan = std::numeric_limits<float>::quiet_NaN();
    std::vector<float> gath(2 * a_plane / 2), win(rows * slot / 2);
    int64_t bad = 0;
    for (int sp = 0; sp < splits; ++sp) {
        const int64_t s0 = sp * per, site_end = (s0 + per < M) ? s0 + per : M;
        for (int64_t site0 = s0; site0 < site_end; site0 += KC) {
            std::fill(gath.begin(), gath.end(), nan);
            std::fill(win.begin(), win.end(), nan);
            for (int mt = 0; mt < 2; ++mt)
                for (int pt = 0; pt < XB_CONV_PRODUCERS; ++pt) {
                    auto emit_a = [&](uint32_t dst, int64_t src) {
                        for (int j = 0; j < 8; ++j) at(gath, mt * a_plane + dst + 2 * j) = src >= 0 ? in[src + j] : 0.f;
                    };
                    auto emit_g = [&](uint32_t, int64_t) {};
                    xb_stage_wgrad(g, tab.data(), pt, mt, site0, site_end, M, 32, 0, emit_a, emit_g);
                }
            const int64_t R0 = site0 / OX;
            for (int j = 0; j < rows; ++j) {
                int b, iy0;
                xb_win_box(g, R0 + j, b, iy0);
                for (int r = 0; r < KH; ++r)
                    for (int u = 0; u < win_w; ++u) {
                        const int iy = iy0 + r, ix = g.dx[0] + u;
                        const bool inside = b < B && iy >= 0 && iy < IH && ix >= 0 && ix < IW;
                        for (int c = 0; c < 8; ++c)
                            at(win, j * slot + (r * win_w + u) * 16 + 2 * c) = inside ? in[(((int64_t)b * IH + iy) * IW + ix) * C + c] : 0.f;
                    }
            }
            for (int wg = 0; wg < 2; ++wg)
                for (int warp = 0; warp < 4; ++warp)
                    for (int lane = 0; lane < 32; ++lane) {
                        const int mi = lane >> 3, lr = lane & 7, m_l = 16 * warp + 8 * (mi & 1);
                        for (int ks = 0; ks < KC / 16; ++ks)
                            for (int r = 0; r < 2; ++r) {
                                const uint32_t ga = r * a_plane + wg * 8192u + (m_l >> 3) * 1024u + (mi >> 1) * 128u + lr * 16u + ks * 256u;
                                const uint32_t wa = xb_win_site_off(g, site0 + 16 * ks + 8 * (mi >> 1) + lr, R0, slot) +
                                                    xb_win_tap_off(g, 128 * r + 64 * wg + m_l, win_w);
                                if (wa + 16 > rows * slot) {
                                    ++bad;
                                    continue;
                                }
                                for (int e = 0; e < 8; ++e)
                                    if (!(at(gath, ga + 2 * e) == at(win, wa + 2 * e))) {
                                        ++bad;
                                        break;
                                    }
                            }
                    }
        }
    }
    return bad;
}

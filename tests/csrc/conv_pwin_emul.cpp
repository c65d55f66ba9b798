// Host emulation of conv_tc_kernel_wgrad_pairs's A operand (conv_tc.cu), built by tests/test_conv_index_pwin.py with g++ (no
// CUDA needed); the index functions are the kernel's own (xuance_b200/csrc/conv_index.h).
#include <cstdint>
#include <limits>
#include <vector>

#include "../../xuance_b200/csrc/conv_index.h"

namespace {
inline float &at(std::vector<float> &smem, uint32_t byte_off) { return smem[byte_off / 2]; }   // one slot per bf16
}

// conv_tc_kernel_wgrad_pairs's A operand against the gathered path's: for every chunk of every split and every 128-row K
// tile, the gathered stage of the three planes is built with xb_stage_wgrad, and the window as the TMA boxes of
// xb_pwin_box fill it: [plane][pair][128 B] per slot, the 16-byte units of each 128-byte row swizzled with bits 7-9 of the
// shared-memory address (the window starts 3 * 8192 bytes into a 1024-byte-aligned stage, after the output-gradient box),
// zero outside the image and past the last image.  Then every ldmatrix row address of every consumer lane, K step and plane
// is formed both ways (conv_tc.cu: the cp.async MN-major lane offset + ks * 256, and xb_sw128 of the window offsets) and
// the 8 values read there compared.  in: [3][B][IH][IW][C].  Returns the number of mismatching rows (-1 on bad input);
// *past_rows counts the rows read whose input row lies past the image's last (IH <= row), which must read as zero.
extern "C" int64_t emul_wgrad_pairs_check(const float *in, int B, int IH, int IW, int C, int OY, int OX, int sy, int sx, int T,
                                          const int8_t *dy, const int8_t *dx, int splits, int64_t *past_rows) {
    XbConvGeom g;
    g.B = B, g.IH = IH, g.IW = IW, g.C = C, g.OY = OY, g.OX = OX, g.sy = sy, g.sx = sx, g.T = T, g.N = 64;
    for (int t = 0; t < XB_CONV_MAX_TAPS; ++t) g.dy[t] = t < T ? dy[t] : 0, g.dx[t] = t < T ? dx[t] : 0;
    xb_geom_finish(g);
    const int KC = XB_CONV_KC, K = T * C, P = 3;
    if (C != 32 || K % XB_CONV_TILE_M != 0 || dx[0] % 2 != 0 || sx % 2 != 0) return -1;
    std::vector<XbUnit> tab(K / 8);
    for (int i = 0; i < K / 8; ++i) tab[i] = xb_unit(g, i);
    const int64_t M = (int64_t)B * OY * OX, per = xb_wgrad_sites_per_split(M, splits), plane = (int64_t)B * IH * IW * C;
    if (per == 0) return -1;
    const int win_w = xb_pwin_width(g), rows = xb_win_rows(g), p0 = dx[0] / 2;
    const uint32_t slot = ((uint32_t)(P * win_w * 128) + 1023u) & ~1023u, a_plane = xb_conv_a_plane_bytes();
    const uint32_t G = P * xb_conv_w_plane_bytes(64), stage = G + rows * slot;
    const float nan = std::numeric_limits<float>::quiet_NaN();
    std::vector<float> gath(P * a_plane / 2), win(stage / 2);
    std::vector<int> past(rows);
    int64_t bad = 0;
    *past_rows = 0;
    for (int sp = 0; sp < splits; ++sp) {
        const int64_t s0 = sp * per, site_end = (s0 + per < M) ? s0 + per : M;
        for (int mt = 0; mt < K / XB_CONV_TILE_M; ++mt)
            for (int64_t site0 = s0; site0 < site_end; site0 += KC) {
                std::fill(gath.begin(), gath.end(), nan);
                std::fill(win.begin(), win.end(), nan);
                for (int pt = 0; pt < XB_CONV_PRODUCERS; ++pt) {
                    auto emit_a = [&](uint32_t dst, int64_t src) {
                        for (int q = 0; q < P; ++q)
                            for (int j = 0; j < 8; ++j) at(gath, q * a_plane + dst + 2 * j) = src >= 0 ? in[q * plane + src + j] : 0.f;
                    };
                    auto emit_g = [&](uint32_t, int64_t) {};
                    xb_stage_wgrad(g, tab.data(), pt, mt, site0, site_end, M, 64, 0, emit_a, emit_g);
                }
                const int64_t R0 = site0 / OX;
                for (int j = 0; j < rows; ++j) {
                    int b, iy;
                    xb_pwin_box(g, R0 + j, mt, b, iy);
                    past[j] = b < B && iy >= IH;
                    for (int q = 0; q < P; ++q)
                        for (int pr = 0; pr < win_w; ++pr) {
                            const uint32_t row_addr = G + j * slot + (q * win_w + pr) * 128;
                            for (int k = 0; k < 128; k += 2) {
                                const int e = k / 2, ix = 2 * (p0 + pr) + e / C, c = e % C;
                                const bool inside = b < B && iy >= 0 && iy < IH && ix >= 0 && ix < IW;
                                const uint32_t dst = row_addr + ((((uint32_t)k >> 4) ^ ((row_addr >> 7) & 7u)) << 4) + (k & 15);
                                at(win, dst) = inside ? in[q * plane + (((int64_t)b * IH + iy) * IW + ix) * C + c] : 0.f;
                            }
                        }
                }
                for (int wg = 0; wg < 2; ++wg)
                    for (int warp = 0; warp < 4; ++warp)
                        for (int lane = 0; lane < 32; ++lane) {
                            const int mi = lane >> 3, lr = lane & 7, m_l = 16 * warp + 8 * (mi & 1);
                            for (int ks = 0; ks < KC / 16; ++ks) {
                                const int64_t s = site0 + 16 * ks + 8 * (mi >> 1) + lr;
                                const uint32_t off = xb_pwin_site_off(g, s, R0, slot) + xb_pwin_tap_off(g, 64 * wg + m_l);
                                const int j = (int)(off / slot);
                                if (j < rows && past[j]) ++*past_rows;
                                for (int q = 0; q < P; ++q) {
                                    const uint32_t ga = q * a_plane + wg * 8192u + (m_l >> 3) * 1024u + (mi >> 1) * 128u + lr * 16u + ks * 256u;
                                    const uint32_t wa = xb_sw128(G + off + q * win_w * 128);
                                    if (wa < G || wa + 16 > stage) {
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
    }
    return bad;
}

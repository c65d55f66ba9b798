// Host view of the staging runs of conv_tc_kernel_dgrad_phases (conv_tc.cu), built by tests/test_conv_index_pairs.py with
// g++ (no CUDA needed); the index functions are the kernel's own (xuance_b200/csrc/conv_index.h).
#include <cstdint>

#include "../../xuance_b200/csrc/conv_index.h"

// For the M tile `tile` of a halo launch over B images of hp raster rows, halo_w positions per row from pixel halo_w0:
// per row phase py (0, 1) and staging slot j < xb_pair_slots(halo_w), the output row the kernel stores (-1: none) and the
// run [lo, hi] of pixels, exactly as the kernel's staging thread computes them.  y1 / oy0 / x1_even / x1_odd are per py.
// Writes 2 * slots entries to each array and returns the slot count.
extern "C" int emul_pair_runs(int B, int hp, int halo_w, int halo_w0, int y0, const int *y1, const int *oy0, const int *x1_even,
                              const int *x1_odd, int out_H, int64_t tile, int64_t *out_row, int *lo, int *hi) {
    const int slots = xb_pair_slots(halo_w);
    const XbDiv div_w = xb_div_make((uint32_t)halo_w), div_hp = xb_div_make((uint32_t)hp);
    const int64_t p0 = tile * XB_CONV_TILE_M;
    const uint32_t R0 = xb_pair_row0(p0, div_w), rows = (uint32_t)B * (uint32_t)hp;
    for (int py = 0; py < 2; ++py)
        for (int j = 0; j < slots; ++j) {
            const int e = py * slots + j;
            out_row[e] = xb_pair_out_row(R0 + j, rows, div_hp, hp, y0, y1[py], oy0[py], out_H);
            if (out_row[e] < 0 || xb_pair_run(p0, R0 + j, halo_w, halo_w0, x1_even[py], x1_odd[py], lo[e], hi[e]) <= 0)
                out_row[e] = -1, lo[e] = 0, hi[e] = -1;
        }
    return slots;
}

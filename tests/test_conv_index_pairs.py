"""CPU: the staging runs of conv2's data gradient by stride-phase pairs (conv_tc_kernel_dgrad_phases,
xuance_b200/csrc/conv_tc.cu; index functions xb_pair_* in conv_index.h).

For every M tile, the output row and pixel run that the kernel's staging thread loads masks for and stores (the host
emulator tests/csrc/conv_pair_emul.cpp calls the kernel's own functions) must be exactly the output elements that the
generic halo epilogue writes from that tile's positions in the two phases of each row phase, enumerated here directly from
the launch geometry.  Over all tiles the runs must cover every real pixel of g1 once and no padding row."""
import ctypes
import os
import subprocess
from collections import defaultdict

import numpy as np
import pytest
import torch.nn as nn

from xuance_b200.torch.utils import tc_conv as tc

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul") / "conv_pair_emul.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", so, os.path.join(HERE, "csrc", "conv_pair_emul.cpp")],
                   check=True)
    lib = ctypes.CDLL(so)
    P, i = ctypes.c_void_p, ctypes.c_int
    lib.emul_pair_runs.argtypes = [i] * 5 + [P] * 4 + [i, ctypes.c_int64, P, P, P]
    lib.emul_pair_runs.restype = i
    return lib


def _plan(B, hw):
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    return tc.BoxNatureCNN(convs, None, (hw, hw, 4))._plan(B)


def _direct(hg, tile):
    """{(py, raster row): set of (output row, pixel)} that the generic epilogue writes from the positions of `tile`."""
    out = defaultdict(set)
    for P in range(128 * tile, min(128 * tile + 128, hg.M)):
        R, hc = divmod(P, hg.halo_w)
        b, y = divmod(R, hg.hp)
        x = hc + hg.halo_w0
        for s, sb in enumerate(hg.subs):
            if 0 <= x <= sb["x1"] and hg.y0 <= y <= sb["y1"]:
                out[(s // 2, R)].add((b * hg.out_H + (y - hg.y0) * hg.oys + sb["oy0"], x * hg.oxs + sb["ox0"]))
    return out


@pytest.mark.parametrize("hw", [84, 88])             # 84: the odd phase one pixel shorter (W1 = 21); 88: equal (W1 = 22)
@pytest.mark.parametrize("B", [1, 2, 3, 7])
def test_pair_runs_are_what_the_generic_epilogue_writes(emul, B, hw):
    P = _plan(B, hw)
    hg = P["h_dg2"]
    assert hg is not None and len(hg.subs) == 4 and (hg.oys, hg.oxs) == (2, 2)
    sb = hg.subs
    i32 = lambda v: np.asarray(v, np.int32)
    y1, oy0 = i32([sb[0]["y1"], sb[2]["y1"]]), i32([sb[0]["oy0"], sb[2]["oy0"]])
    x1e, x1o = i32([sb[0]["x1"], sb[2]["x1"]]), i32([sb[1]["x1"], sb[3]["x1"]])
    slots = (128 - 2 + hg.halo_w) // hg.halo_w + 1
    orow, lo, hi = np.zeros(2 * slots, np.int64), np.zeros(2 * slots, np.int32), np.zeros(2 * slots, np.int32)
    written = np.zeros((B * P["hp1"], P["W1"]), np.int32)
    tiles = -(-hg.M // 128)
    for t in range(tiles):
        n = emul.emul_pair_runs(B, hg.hp, hg.halo_w, hg.halo_w0, hg.y0, y1.ctypes.data, oy0.ctypes.data, x1e.ctypes.data,
                                x1o.ctypes.data, hg.out_H, t, orow.ctypes.data, lo.ctypes.data, hi.ctypes.data)
        assert n == slots
        want = _direct(hg, t)
        R0 = 128 * t // hg.halo_w
        assert all(0 <= R - R0 < slots for _, R in want), (t, sorted(want))
        for py in range(2):
            for j in range(slots):
                e = py * slots + j
                got = set() if orow[e] < 0 else {(int(orow[e]), x) for x in range(lo[e], hi[e] + 1)}
                assert got == want.get((py, R0 + j), set()), (B, hw, t, py, j, int(orow[e]), int(lo[e]), int(hi[e]))
                if orow[e] >= 0:
                    written[orow[e], lo[e]:hi[e] + 1] += 1
    real = np.zeros_like(written, dtype=bool).reshape(B, P["hp1"], P["W1"])
    real[:, P["off1"]:P["off1"] + P["H1"]] = True
    assert (written[real.reshape(written.shape)] == 1).all()
    assert (written[~real.reshape(written.shape)] == 0).all()

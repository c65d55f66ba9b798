"""CPU: addressing of the pixel-pair windows that conv2's weight gradient reads its A operand from
(conv_tc_kernel_wgrad_pairs, xuance_b200/csrc/conv_tc.cu; index functions xb_pwin_* and xb_sw128 in conv_index.h).

The host emulator (tests/csrc/conv_pwin_emul.cpp) stages every chunk and K tile the way the gathered cp.async path does
and fills the window the way the swizzled TMA boxes do, then forms every consumer lane's ldmatrix row address both ways and
compares the 16 bytes read there, for all three planes: the window path must see exactly the values the gathered path
stages, zeros included.  The input has no zero anywhere, so a row past an image's last one reads as zero only if it is
the zero fill, not the next image's first row."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn as nn

from xuance_b200.torch.utils import tc_conv as tc

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul") / "conv_pwin_emul.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", so, os.path.join(HERE, "csrc", "conv_pwin_emul.cpp")],
                   check=True)
    lib = ctypes.CDLL(so)
    P, i = ctypes.c_void_p, ctypes.c_int
    lib.emul_wgrad_pairs_check.argtypes = [P] + [i] * 9 + [P, P, i, P]
    lib.emul_wgrad_pairs_check.restype = ctypes.c_int64
    return lib


def _wg2(B):
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    return tc.BoxNatureCNN(convs, None, (84, 84, 4))._plan(B)["wg2"]


def _single_chunk_tail(M):
    """A split count whose last run of sites is one chunk of at most 64 sites."""
    for s in range(2, M // 64 + 2):
        per = -(-(-(-M // s)) // 64) * 64
        if (s - 1) * per < M and M - (s - 1) * per <= 64:
            return s
    raise AssertionError(M)


@pytest.mark.parametrize("B", [1, 3, 16])
def test_pair_window_rows_read_what_the_gather_stages(emul, B):
    """conv2's weight-gradient geometry over act1 (12 grid rows of 10 sites per image, 24 input rows of 22 pixels): chunks
    that start anywhere in a grid row, cross image boundaries (B > 1), read input rows 24 and 25 of an image (grid row 11,
    tap rows 2 and 3) and run past the last site."""
    g = _wg2(B)
    assert (g.C, g.K, g.sx, g.OX, g.OY, g.IH, g.IW) == (32, 512, 2, 10, 12, 24, 22)
    x = torch.randint(1, 256, (3, g.B, g.IH, g.IW, g.C)).float().contiguous()     # no zero: a zero must come from padding
    dy, dx = np.asarray(g.dy, np.int8), np.asarray(g.dx, np.int8)
    for splits in sorted({1, tc.wgrad_splits(g.M, g.K), _single_chunk_tail(g.M)}):
        past = ctypes.c_int64(0)
        bad = emul.emul_wgrad_pairs_check(x.data_ptr(), g.B, g.IH, g.IW, g.C, g.OY, g.OX, g.sy, g.sx, g.T, dy.ctypes.data,
                                          dx.ctypes.data, splits, ctypes.byref(past))
        assert bad == 0, "splits=%d: %d ldmatrix rows differ" % (splits, bad)
        assert past.value > 0, "no lane read a row past an image's last"

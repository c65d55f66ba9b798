"""CPU: addressing of the input windows that conv1's weight gradient reads its A operand from (conv_tc_kernel_wgrad_win,
xuance_b200/csrc/conv_tc.cu; index functions xb_win_* in conv_index.h).

The host emulator (tests/csrc/conv_win_emul.cpp) stages every chunk the way the gathered cp.async path does and fills the
window the way the TMA boxes do, then forms every consumer lane's ldmatrix row address both ways and compares the 16 bytes
read there: the window path must see exactly the values the gathered path stages, zeros included."""
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
    so = str(tmp_path_factory.mktemp("emul") / "conv_win_emul.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", so, os.path.join(HERE, "csrc", "conv_win_emul.cpp")],
                   check=True)
    lib = ctypes.CDLL(so)
    P, i = ctypes.c_void_p, ctypes.c_int
    lib.emul_wgrad_win_check.argtypes = [P] + [i] * 9 + [P, P, i]
    lib.emul_wgrad_win_check.restype = ctypes.c_int64
    return lib


def _wg1(B):
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    return tc.BoxNatureCNN(convs, None, (84, 84, 4))._plan(B)["wg1"]


def _single_chunk_tail(M):
    """A split count whose last run of sites is one chunk of at most 64 sites."""
    for s in range(2, M // 64 + 2):
        per = -(-(-(-M // s)) // 64) * 64
        if (s - 1) * per < M and M - (s - 1) * per <= 64:
            return s
    raise AssertionError(M)


@pytest.mark.parametrize("B", [1, 3])
def test_window_rows_read_what_the_gather_stages(emul, B):
    """conv1's weight-gradient geometry over the padded act1 grid (24 rows of 21 sites per image, rows 0-2 garbage): chunks
    that start anywhere in a grid row, cross image boundaries (B = 3) and run past the last site."""
    g = _wg1(B)
    assert (g.C, g.K, g.sx, g.OX) == (8, 256, 2, 21)
    x = torch.randint(1, 256, (g.B, g.IH, g.IW, g.C)).float().contiguous()     # no zero pixels: a zero must come from padding
    dy, dx = np.asarray(g.dy, np.int8), np.asarray(g.dx, np.int8)
    for splits in sorted({1, tc.wgrad_splits(g.M, g.K), _single_chunk_tail(g.M)}):
        bad = emul.emul_wgrad_win_check(x.data_ptr(), g.B, g.IH, g.IW, g.C, g.OY, g.OX, g.sy, g.sx, g.T, dy.ctypes.data,
                                        dx.ctypes.data, splits)
        assert bad == 0, "splits=%d: %d ldmatrix rows differ" % (splits, bad)

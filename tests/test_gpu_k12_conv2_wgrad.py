"""GPU: conv2's weight gradient from TMA pixel-pair windows (conv_tc_kernel_wgrad_pairs, taken by xb_wgrad_gather_tc for
three planes, 32 input channels read as pixel pairs, a 4 x 4 tap rectangle, N = 64) against the gathered cp.async path
(XB_K12_TMA=0 in a subprocess), which sums the same products into the same accumulators in the same order: the partials
must be equal bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the reference run: the same inputs through the gathered path only
_REF = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
from xuance_b200.torch.utils import tc_conv as tc
d = torch.load(sys.argv[2], weights_only=False)
out = {}
for key, (geom, splits) in d["cases"].items():
    out[key] = tc.wgrad_gather(d["x"][geom.B].cuda(), d["g"][geom.B].cuda(), geom, splits).cpu()
torch.save(out, sys.argv[3])
"""


def _wg2(B):
    from xuance_b200.torch.utils import tc_conv as tc
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    return tc.BoxNatureCNN(convs, None, (84, 84, 4))._plan(B)["wg2"]


def _single_chunk_tail(M):
    for s in range(2, M // 64 + 2):
        per = -(-(-(-M // s)) // 64) * 64
        if (s - 1) * per < M and M - (s - 1) * per <= 64:
            return s
    raise AssertionError(M)


def _inputs(B, seed):
    """Every input row non-zero, the padding rows of act1's layout included: a window row read from the next image instead
    of the zero fill would change the partials."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    geom = _wg2(B)
    x = torch.randn((3, B * geom.IH, geom.IW, geom.C), device=DEV, generator=g).to(torch.bfloat16)
    gr = torch.randn((3, geom.M, 64), device=DEV, generator=g).to(torch.bfloat16)
    return geom, x, gr


def _bits(t):
    return t.contiguous().view(torch.int32)


def test_partials_bitwise_equal_to_gathered_path(tmp_path):
    from xuance_b200.torch.utils import tc_conv as tc
    cases, xs, gs, got = {}, {}, {}, {}
    for B in (1, 3, 16, 300):
        geom, x, gr = _inputs(B, B)
        xs[B], gs[B] = x.cpu(), gr.cpu()
        for splits in sorted({tc.wgrad_splits(geom.M, geom.K), _single_chunk_tail(geom.M)}):
            key = "B%d_s%d" % (B, splits)
            cases[key] = (geom, splits)
            got[key] = tc.wgrad_gather(x, gr, geom, splits)
            again = tc.wgrad_gather(x, gr, geom, splits)
            assert torch.equal(_bits(got[key]), _bits(again)), key                 # two launches agree bit for bit
    src, dst = tmp_path / "in.pt", tmp_path / "ref.pt"
    torch.save(dict(cases=cases, x=xs, g=gs), src)
    env = dict(os.environ, XB_K12_TMA="0")
    res = subprocess.run([sys.executable, "-c", _REF, ROOT, str(src), str(dst)], env=env, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    ref = torch.load(dst, weights_only=False)
    for key in cases:
        a, b = got[key].cpu(), ref[key]
        diff = (a.double() - b.double()).abs().max().item()
        assert torch.equal(_bits(a), _bits(b)), "%s: largest difference %g" % (key, diff)


def test_padded_geometry_against_float64_autograd():
    """dW2 over act1's padded layout (real rows 3 .. 23, real pixels 1 .. 21) and the padded output grid (real rows 1 .. 10
    of 12) vs autograd of the unpadded convolution."""
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(5)
    B, N = 16, 64
    geom = _wg2(B)
    a1 = torch.rand((B, 21, 21, 32), device=DEV, dtype=torch.float64)
    w = (torch.randn(N, 32, 4, 4, device=DEV, dtype=torch.float64) / 16).requires_grad_(True)
    y = F.conv2d(a1.permute(0, 3, 1, 2), w, stride=2, padding=1)
    gy = torch.randn(y.shape, device=DEV, dtype=torch.float64) / np.sqrt(100 * B)
    (want,) = torch.autograd.grad(y, w, gy)
    xpad = torch.zeros((B, geom.IH, geom.IW, 32), device=DEV)
    xpad[:, 3:24, 1:22] = a1.float()
    gpad = torch.zeros((B, geom.OY, geom.OX, N), device=DEV)
    gpad[:, 1:11] = gy.permute(0, 2, 3, 1).float()
    x_pl = tc.split_bf16(xpad.reshape(-1).contiguous(), 3).view(3, B * geom.IH, geom.IW, 32)
    g_pl = tc.split_bf16(gpad.reshape(geom.M, N).contiguous(), 3)
    dw = tc.wgrad_reduce(tc.wgrad_gather(x_pl, g_pl, geom, tc.wgrad_splits(geom.M, geom.K)), N, 32, 4, 4)
    np.testing.assert_allclose(dw.cpu().numpy(), want.cpu().numpy(), rtol=0, atol=2e-5 * max(1.0, float(want.abs().max())))

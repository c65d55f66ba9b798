"""GPU: conv1's weight gradient from TMA input windows (conv_tc_kernel_wgrad_win, taken by xb_wgrad_gather_tc for one raw
pixel plane, 4 channels, N = 32) against the gathered cp.async path (XB_K12_TMA=0 in a subprocess), which sums the same
products into the same accumulators in the same order: the partials must be equal bit for bit."""
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


def _wg1(B):
    from xuance_b200.torch.utils import tc_conv as tc
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    return tc.BoxNatureCNN(convs, None, (84, 84, 4))._plan(B)["wg1"]


def _single_chunk_tail(M):
    for s in range(2, M // 64 + 2):
        per = -(-(-(-M // s)) // 64) * 64
        if (s - 1) * per < M and M - (s - 1) * per <= 64:
            return s
    raise AssertionError(M)


def _inputs(B, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    geom = _wg1(B)
    x = torch.randint(0, 256, (1, B, 84, 84, 4), device=DEV, generator=g).to(torch.bfloat16)
    gr = torch.randn((3, geom.M, 32), device=DEV, generator=g).to(torch.bfloat16)
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
    """dW1 over the padded act1 grid (gradient zero on its garbage rows) vs autograd of the unpadded convolution."""
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(3)
    B, N = 16, 32
    geom = _wg1(B)
    obs = torch.randint(0, 256, (B, 84, 84, 4), dtype=torch.uint8, device=DEV)
    w = (torch.randn(N, 4, 8, 8, device=DEV, dtype=torch.float64) / 16).requires_grad_(True)
    y = F.conv2d((obs.double() / 255.0).permute(0, 3, 1, 2), w, stride=4, padding=2)
    gy = torch.randn(y.shape, device=DEV) / np.sqrt(441 * B)
    (want,) = torch.autograd.grad(y, w, gy.double())
    gpad = torch.zeros((B, geom.OY, geom.OX, N), device=DEV)
    gpad[:, geom.OY - 21:] = gy.permute(0, 2, 3, 1)                    # real act1 rows are the last 21 of the padded grid
    raw = obs.to(torch.bfloat16).unsqueeze(0)
    g_pl = tc.split_bf16(gpad.reshape(geom.M, N).contiguous(), 3)
    dw = tc.wgrad_reduce(tc.wgrad_gather(raw, g_pl, geom, tc.wgrad_splits(geom.M, geom.K)), N, 4, 8, 8, scale=1.0 / 255.0)
    np.testing.assert_allclose(dw.cpu().numpy(), want.cpu().numpy(), rtol=0, atol=3e-6 * max(1.0, float(want.abs().max())))

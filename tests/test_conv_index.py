"""CPU: index arithmetic and layer geometry of the EXPERIMENTAL tensor-core conv path (K12, xuance_b200/csrc/conv_tc.cu).

The kernel cannot run here, so its data movement is emulated on the host WITH THE KERNEL'S OWN index functions
(xuance_b200/csrc/conv_index.h is compiled into tests/csrc/conv_emul.cpp by g++): units are staged into an emulated
shared-memory image, read back the way the wgmma descriptors address it, and the result is compared with torch's fp64
convolution / autograd on the un-split operands - which also checks the split-bf16 numerics claim (three products of
hi/lo bf16 pairs reproduce the fp32 result to ~1e-5)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.tc_numerics import split_planes
from xuance_b200.torch.utils import tc_conv as tc

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emul():
    src, so = os.path.join(HERE, "csrc", "conv_emul.cpp"), os.path.join(HERE, "csrc", "_conv_emul.so")
    hdr = os.path.join(HERE, "..", "xuance_b200", "csrc", "conv_index.h")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", so, src], check=True)
    lib = ctypes.CDLL(so)
    P, i, l = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    lib.emul_gemm_gather.argtypes = [i, i, P, l, P, l] + [i] * 9 + [P, P] + [i] * 8 + [l, i, i, P]
    lib.emul_gemm_gather.restype = i
    lib.emul_pack_weight.argtypes = [P, i, i, i, i, P]
    lib.emul_wgrad.argtypes = [i, i, P, l, P, l, l] + [i] * 9 + [P, P] + [i] * 4 + [P]
    lib.emul_wgrad.restype = i
    lib.emul_wgrad_reduce.argtypes = [P, i, i, i, i, i, ctypes.c_double, P]
    return lib


def _split(x, planes=2):
    """float -> float32 [planes, ...] of bf16-representable values (oracle/tc_numerics.py: what xb_split_bf16 and the
    kernel epilogues produce)."""
    return split_planes(x, planes)


def _run(lib, geom, x_nhwc, w_mat, out, out_ld, out_c0=0, stages=2, planes=2, planes_a=None):
    """x_nhwc: float64 tensor viewed as the geometry's [B, IH, IW, C]; w_mat float64 [N, K]; out float64 [rows, out_ld].
    ``planes_a``: planes of the A operand (default ``planes``; 1 = values that one bf16 holds exactly)."""
    pa = planes if planes_a is None else planes_a
    xp, wp = _split(x_nhwc, pa), _split(w_mat, planes)
    N, K = w_mat.shape
    assert K == geom.K and xp[0].numel() == geom.B * geom.IH * geom.IW * geom.C
    dy, dx = np.asarray(geom.dy, np.int8), np.asarray(geom.dx, np.int8)
    rc = lib.emul_gemm_gather(pa, planes, xp.data_ptr(), xp.stride(0), wp.data_ptr(), wp.stride(0), geom.B, geom.IH, geom.IW,
                              geom.C, geom.OY, geom.OX, geom.sy, geom.sx, geom.T, dy.ctypes.data, dx.ctypes.data, N,
                              tc.n_tile_for(N, planes), geom.out_H, geom.out_W, geom.oys, geom.oxs, geom.oy0, geom.ox0, out_ld,
                              out_c0, stages, out.data_ptr())
    assert rc == 0


def _pack(lib, w):
    N, C, KH, KW = w.shape
    wf = w.float().contiguous()
    packed = torch.empty((N, KH * KW * C), dtype=torch.float32)
    lib.emul_pack_weight(wf.data_ptr(), N, C, KH, KW, packed.data_ptr())
    ref = w.permute(0, 2, 3, 1).reshape(N, -1).float()         # (kh, kw, c) column order
    assert torch.equal(packed, ref)
    return packed.double()


TOL = dict(rtol=0, atol=4e-5)     # |x - hi - lo| <= 2^-17 |x| per operand; sums of <= 6400 products of O(1) values / sqrt(K)


@pytest.mark.parametrize("planes", [2, 3])
@pytest.mark.parametrize("name,B,H,W,C,N,k,s", [("conv1", 2, 84, 84, 4, 32, 8, 4), ("conv2", 2, 21, 21, 32, 64, 4, 2),
                                                ("conv3", 3, 10, 10, 64, 64, 3, 1), ("odd", 1, 13, 9, 8, 32, 4, 2)])
def test_forward_conv_layers(emul, name, B, H, W, C, N, k, s, planes):
    """The three NatureCNN convolutions with the reference's padding rule (k - s)//2 (layers.py:46), NHWC input."""
    torch.manual_seed(len(name))
    pad = (k - s) // 2
    x = torch.rand(B, C, H, W, dtype=torch.float64)                       # observations / 255 live in [0, 1]
    w = torch.randn(N, C, k, k, dtype=torch.float64) / np.sqrt(C * k * k)
    g = tc.conv_forward_geometry(B, H, W, C, k, k, s, pad)
    assert g.K == C * k * k and (g.fold == 2) == (C == 4)
    out = torch.full((g.M, N), float("nan"), dtype=torch.float64)
    _run(emul, g, x.permute(0, 2, 3, 1).contiguous(), _pack(emul, w), out, N, planes=planes)
    want = F.conv2d(x, w, stride=s, padding=pad).permute(0, 2, 3, 1).reshape(g.M, N)
    # 2 planes: operands exact to 2^-17; 3 planes: to 2^-24 (the float32 inputs themselves are only exact to 2^-24)
    np.testing.assert_allclose(out.numpy(), want.numpy(), rtol=0, atol=4e-5 if planes == 2 else 6e-7)


def test_linear_layer_with_column_split_and_row_tail(emul):
    """Linear(6400 -> 512) over the NHWC-flattened conv3 output: N = 512 runs as column tiles of 128 (two planes) inside one
    call and as two 256-column calls; 130 rows leave a 2-row tail tile.  The reference flattens NCHW (cnn.py:92), so the
    packed weight permutes its columns to (h, w, c)."""
    torch.manual_seed(0)
    Bn, Cc, Hh, Ww, N = 130, 64, 10, 10, 512
    feat = torch.rand(Bn, Cc, Hh, Ww, dtype=torch.float64)
    w = torch.randn(N, Cc * Hh * Ww, dtype=torch.float64) / 80.0
    packed = _pack(emul, w.reshape(N, Cc, Hh, Ww))                         # columns (h, w, c)
    g = tc.linear_geometry(Bn, Cc * Hh * Ww)
    out = torch.full((Bn, N), float("nan"), dtype=torch.float64)
    x_nhwc = feat.permute(0, 2, 3, 1).reshape(Bn, 1, 1, -1).contiguous()
    for c0 in (0, 256):
        _run(emul, g, x_nhwc, packed[c0:c0 + 256].contiguous(), out, N, out_c0=c0, stages=2)
    want = feat.reshape(Bn, -1) @ w.t()
    np.testing.assert_allclose(out.numpy(), want.numpy(), **TOL)
    out.fill_(float("nan"))
    _run(emul, g, x_nhwc, packed, out, N, stages=3, planes=3)                     # 8 column tiles of 64, three planes
    np.testing.assert_allclose(out.numpy(), want.numpy(), rtol=0, atol=2e-6)


def test_raw_uint8_plane_first_layer(emul):
    """conv1 on ONE exact plane of raw uint8 pixel values against three weight planes carrying the 1/255."""
    torch.manual_seed(5)
    B, H, W, C, N, k, s = 2, 84, 84, 4, 32, 8, 4
    obs = torch.randint(0, 256, (B, H, W, C), dtype=torch.uint8)
    w = torch.randn(N, C, k, k, dtype=torch.float64) / np.sqrt(C * k * k)
    g = tc.conv_forward_geometry(B, H, W, C, k, k, s, 2)
    out = torch.full((g.M, N), float("nan"), dtype=torch.float64)
    w_scaled = (w.float() * np.float32(1.0 / 255.0)).double()
    _run(emul, g, obs.double(), _pack(emul, w_scaled), out, N, planes=3, planes_a=1)
    want = F.conv2d((obs.double() / 255.0).permute(0, 3, 1, 2), w, stride=s, padding=2).permute(0, 2, 3, 1).reshape(g.M, N)
    np.testing.assert_allclose(out.numpy(), want.numpy(), rtol=0, atol=6e-7)


@pytest.mark.parametrize("name,B,H,W,C,N,k,s", [("conv3", 2, 10, 10, 64, 64, 3, 1), ("conv2", 2, 21, 21, 32, 64, 4, 2),
                                                ("s4", 1, 20, 20, 32, 32, 8, 4)])
def test_data_gradient_phases(emul, name, B, H, W, C, N, k, s):
    """grad_input of a convolution as one gathered GEMM per stride phase over the output gradient, vs autograd."""
    torch.manual_seed(1)
    pad = (k - s) // 2
    x = torch.randn(B, C, H, W, dtype=torch.float64, requires_grad=True)
    w = torch.randn(N, C, k, k, dtype=torch.float64) / np.sqrt(N * k * k / (s * s))
    y = F.conv2d(x, w, stride=s, padding=pad)
    gy = torch.randn_like(y)
    (want,) = torch.autograd.grad(y, x, gy)
    gy_nhwc = gy.permute(0, 2, 3, 1).contiguous()
    out = torch.full((B * H * W, C), float("nan"), dtype=torch.float64)
    phases = tc.conv_dgrad_geometries(B, H, W, C, k, k, s, pad, N)
    assert len(phases) == s * s and sum(len(t) for _, t in phases) == k * k
    for g, taps in phases:
        _run(emul, g, gy_nhwc, tc.dgrad_weight_matrix(w, taps), out, C)
    np.testing.assert_allclose(out.reshape(B, H, W, C).permute(0, 3, 1, 2).numpy(), want.numpy(), **TOL)


@pytest.mark.parametrize("name,B,H,W,C,N,k,s,splits", [("conv1", 2, 84, 84, 4, 32, 8, 4, 3), ("conv2", 4, 21, 21, 32, 64, 4, 2, 3),
                                                       ("conv3", 3, 10, 10, 64, 64, 3, 1, 2), ("conv3_1split", 1, 10, 10, 64, 64, 3, 1, 1)])
def test_weight_gradient(emul, name, B, H, W, C, N, k, s, splits):
    """grad_weight as the MN-major gathered GEMM (split over sites, then reduced into torch's [N, C, KH, KW]) vs autograd.
    conv3 has K = 576 = 4.5 column tiles (a half-empty tile); conv1 runs on the pixel-folded view."""
    torch.manual_seed(2)
    pad = (k - s) // 2
    x = torch.rand(B, C, H, W, dtype=torch.float64)
    w = (torch.randn(N, C, k, k, dtype=torch.float64) / np.sqrt(C * k * k)).requires_grad_(True)
    y = F.conv2d(x, w, stride=s, padding=pad)
    gy = torch.randn_like(y) / np.sqrt(y[0, 0].numel())
    (want,) = torch.autograd.grad(y, w, gy)
    g = tc.conv_forward_geometry(B, H, W, C, k, k, s, pad)             # the weight gradient gathers like the forward
    planes = 3 if name == "conv3" else 2
    xp = _split(x.permute(0, 2, 3, 1).contiguous(), planes)
    gp = _split(gy.permute(0, 2, 3, 1).reshape(g.M, N).contiguous(), planes)
    partials = torch.full((splits, g.K, N), float("nan"), dtype=torch.float64)
    dy, dx = np.asarray(g.dy, np.int8), np.asarray(g.dx, np.int8)
    rc = emul.emul_wgrad(planes, planes, xp.data_ptr(), xp.stride(0), gp.data_ptr(), gp.stride(0), N, g.B, g.IH, g.IW, g.C, g.OY,
                         g.OX, g.sy, g.sx, g.T, dy.ctypes.data, dx.ctypes.data, N, tc.n_tile_for(N, planes), splits, 2,
                         partials.data_ptr())
    assert rc == 0 and not torch.isnan(partials).any()
    dw = torch.full((N, C, k, k), float("nan"), dtype=torch.float64)
    emul.emul_wgrad_reduce(partials.data_ptr(), splits, N, C, k, k, 1.0, dw.data_ptr())
    np.testing.assert_allclose(dw.numpy(), want.numpy(), **TOL)


def test_linear_weight_gradient(emul):
    """dW of Linear(6400 -> 128): sites = batch rows, one tap, 50 row tiles x 2 column tiles of 64 of a gradient matrix whose
    rows are 128 elements apart."""
    torch.manual_seed(3)
    Bn, K, N = 70, 6400, 128
    x = torch.rand(Bn, K, dtype=torch.float64)
    gy = torch.randn(Bn, N, dtype=torch.float64) / 8
    g = tc.linear_geometry(Bn, K)
    xp, gp = _split(x), _split(gy)
    partials = torch.full((2, K, N), float("nan"), dtype=torch.float64)
    dy, dx = np.zeros(1, np.int8), np.zeros(1, np.int8)
    rc = emul.emul_wgrad(2, 2, xp.data_ptr(), xp.stride(0), gp.data_ptr(), gp.stride(0), N, g.B, 1, 1, K, 1, 1, 1, 1, 1,
                         dy.ctypes.data, dx.ctypes.data, N, 64, 2, 2, partials.data_ptr())
    assert rc == 0 and not torch.isnan(partials).any()
    np.testing.assert_allclose(partials.sum(0).t().numpy(), (gy.t() @ x).numpy(), **TOL)


def test_fast_division_is_exact(emul):
    """xb_div: every divisor the layers use (sites per image, grid width) and awkward ones, over ranges of n < 2^31."""
    emul.emul_div_check.restype = ctypes.c_int64
    emul.emul_div_check.argtypes = [ctypes.c_uint32] * 3
    for d in (1, 2, 3, 7, 10, 21, 100, 441, 484, 144, 6400, 12345, 65537, 1 << 20, (1 << 31) - 1):
        assert emul.emul_div_check(d, 0, 200000) == 0, d
        assert emul.emul_div_check(d, 3612672 - 1000, 3612672 + 1000) == 0, d


def test_wgrad_split_rule():
    """xb_wgrad_sites_per_split (mirrored here): runs are multiples of 64 sites and never empty."""
    def per(M, splits):
        p = -(-M // splits)
        p = -(-p // 64) * 64
        return 0 if (splits - 1) * p >= M else p
    assert per(882, 3) == 320 and per(200, 5) == 0 and per(64, 1) == 64 and per(8192 * 100, 37) % 64 == 0


class EmulBackend:
    """``TensorCoreNatureCNN`` backend that runs every K12 launch through the host emulator (CPU float32 tensors holding
    bf16-representable values stand in for the bf16 planes).  The epilogue (bias, ReLU, mask, output formats) is restated
    here; staging, operand layouts and work decomposition are the kernel's own code (conv_index.h)."""

    def __init__(self, lib, planes=2):
        self.lib, self.planes = lib, planes

    def split(self, x):
        return _split(x, self.planes)

    def pack_weight(self, w4d, scale=1.0):
        N = w4d.shape[0]
        return _split(w4d.float().permute(0, 2, 3, 1).reshape(N, -1) * np.float32(scale), self.planes)

    def empty_planes(self, shape, like):
        return torch.full((self.planes,) + tuple(shape), float("nan"))

    def empty_f32(self, shape, like):
        return torch.full(shape, float("nan"))

    def to_float(self, pl):
        return pl.sum(0)

    def colsum(self, g_pl):
        return g_pl.double().sum(dim=(0, 1)).float()

    def gemm(self, x_pl, w_pl, geom, bias=None, relu=False, out_f32=None, out_pl=None, out_ld=None, out_c0=0, mask=None):
        P, N = w_pl.shape[0], w_pl.shape[1]
        PA = x_pl.shape[0]
        out_ld = N if out_ld is None else out_ld
        rows = geom.B * geom.out_H * geom.out_W
        tmp = torch.full((rows, out_ld), float("nan"), dtype=torch.float64)
        x_pl, w_pl = x_pl.contiguous(), w_pl.contiguous()
        dy, dx = np.asarray(geom.dy, np.int8), np.asarray(geom.dx, np.int8)
        rc = self.lib.emul_gemm_gather(PA, P, x_pl.data_ptr(), x_pl.stride(0), w_pl.data_ptr(), w_pl.stride(0), geom.B,
                                       geom.IH, geom.IW, geom.C, geom.OY, geom.OX, geom.sy, geom.sx, geom.T, dy.ctypes.data,
                                       dx.ctypes.data, N, tc.n_tile_for(N, P), geom.out_H, geom.out_W, geom.oys, geom.oxs,
                                       geom.oy0, geom.ox0, out_ld, out_c0, 2, tmp.data_ptr())
        assert rc == 0
        blk = tmp[:, out_c0:out_c0 + N]
        written = ~torch.isnan(blk[:, 0])
        assert int(written.sum()) == geom.M
        v = blk[written]
        if bias is not None:
            v = v + bias.double()
        if relu:
            v = v.clamp_min(0)
        if mask is not None:
            v = torch.where(mask.reshape(rows, out_ld)[written, out_c0:out_c0 + N] > 0, v, torch.zeros_like(v))
        v = v.float()
        if out_f32 is not None:
            out_f32.view(rows, out_ld)[written, out_c0:out_c0 + N] = v
        if out_pl is not None:
            Po = out_pl.shape[0]
            out_pl.view(Po, rows, out_ld)[:, written, out_c0:out_c0 + N] = _split(v, Po)

    def wgrad(self, x_pl, g_pl, geom, N, C, KH, KW, scale=1.0):
        P, PA = g_pl.shape[0], x_pl.shape[0]
        splits = 2 if geom.M > 128 else 1
        partials = torch.full((splits, geom.K, N), float("nan"), dtype=torch.float64)
        dy, dx = np.asarray(geom.dy, np.int8), np.asarray(geom.dx, np.int8)
        x_pl, g_pl = x_pl.contiguous(), g_pl.contiguous()
        rc = self.lib.emul_wgrad(PA, P, x_pl.data_ptr(), x_pl.stride(0), g_pl.data_ptr(), g_pl.stride(0), g_pl.stride(1), geom.B,
                                 geom.IH, geom.IW, geom.C, geom.OY, geom.OX, geom.sy, geom.sx, geom.T, dy.ctypes.data,
                                 dx.ctypes.data, N, tc.n_tile_for(N, P), splits, 2, partials.data_ptr())
        assert rc == 0 and not torch.isnan(partials).any()
        dw = torch.full((N, C, KH, KW), float("nan"), dtype=torch.float64)
        self.lib.emul_wgrad_reduce(partials.data_ptr(), splits, N, C, KH, KW, float(np.float32(scale)), dw.data_ptr())
        return dw.float()


@pytest.mark.parametrize("planes", [2, 3])
def test_nature_cnn_forward_backward_orchestration(emul, planes):
    """The whole encoder (3 convs + Linear, cnn.py:84-101) forward and backward through TensorCoreNatureCNN with the
    emulated backend vs torch autograd in float64: layer chaining, NHWC <-> NCHW-flatten weight permutation, ReLU masks in
    the data-gradient epilogues, stride-phase data gradients, column-split Linear (320 = 256 + 64 outputs)."""
    import torch.nn as nn
    torch.manual_seed(7)
    B, hidden = 2, 320
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    fc = nn.Linear(6400, hidden)
    for m in convs + [fc]:
        nn.init.orthogonal_(m.weight, gain=np.sqrt(2))
        nn.init.uniform_(m.bias, -0.05, 0.05)
    obs = torch.randint(0, 256, (B, 84, 84, 4), dtype=torch.uint8)
    x = obs.float() / 255.0
    R = torch.randn(B, hidden)
    # reference: torch autograd in float64, NCHW
    ref = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1),
           nn.Linear(6400, hidden)]
    for r, m in zip(ref, convs + [fc]):
        r.load_state_dict(m.state_dict())
        r.double()
    h = x.double().permute(0, 3, 1, 2)
    for r in ref[:3]:
        h = torch.relu(r(h))
    z_ref = torch.relu(ref[3](h.flatten(1)))
    (z_ref * R.double()).sum().backward()
    # K12 path on the emulator
    enc = tc.TensorCoreNatureCNN(convs, fc, (84, 84, 4), backend=EmulBackend(emul, planes))
    # three planes: the raw uint8 pixels as ONE exact plane (1/255 in the first layer's weights); two planes: x/255 split
    x_in = _split(obs.float(), 1) if planes == 3 else _split(x, planes)
    z = tc.tc_encode(enc, x_in, B)
    np.testing.assert_allclose(z.detach().numpy(), z_ref.detach().numpy(), rtol=1e-4, atol=1e-4)
    (z * R).sum().backward()
    for (m, r), name in zip(zip(convs + [fc], ref), ("conv1", "conv2", "conv3", "fc")):
        scale = float(r.weight.grad.abs().max())
        np.testing.assert_allclose(m.weight.grad.numpy(), r.weight.grad.numpy(), rtol=0, atol=2e-4 * scale, err_msg=name)
        np.testing.assert_allclose(m.bias.grad.numpy(), r.bias.grad.numpy(), rtol=0,
                                   atol=2e-4 * float(r.bias.grad.abs().max()), err_msg=name + ".bias")


def test_pooled_conv_stack_orchestration(emul):
    """Basic_CNN's shape (cnn.py:11-50): three convolutions, global max pool, no hidden layer - the encoder of the DQN
    family.  The pooled gradient reaches the K12 backward as a sparse [sites, C] array."""
    import torch.nn as nn
    torch.manual_seed(9)
    B = 2
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    ref = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    for r, m in zip(ref, convs):
        r.load_state_dict(m.state_dict())
        r.double()
    x = torch.randint(0, 256, (B, 84, 84, 4), dtype=torch.uint8).float() / 255.0
    R = torch.randn(B, 64)
    h = x.double().permute(0, 3, 1, 2)
    for r in ref:
        h = torch.relu(r(h))
    feat_ref = torch.amax(h, dim=(2, 3))
    (feat_ref * R.double()).sum().backward()
    enc = tc.TensorCoreNatureCNN(convs, None, (84, 84, 4), backend=EmulBackend(emul, 3))
    z = tc.tc_encode(enc, _split(x, 3), B)
    feat = z.view(B, -1, 64).amax(dim=1)
    np.testing.assert_allclose(feat.detach().numpy(), feat_ref.detach().numpy(), rtol=1e-5, atol=1e-6)
    (feat * R).sum().backward()
    for m, r in zip(convs, ref):
        np.testing.assert_allclose(m.weight.grad.numpy(), r.weight.grad.numpy(), rtol=0,
                                   atol=2e-5 * float(r.weight.grad.abs().max()))
        np.testing.assert_allclose(m.bias.grad.numpy(), r.bias.grad.numpy(), rtol=0,
                                   atol=2e-5 * float(r.bias.grad.abs().max()))

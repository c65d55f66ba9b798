"""Host side of K12 (``xb_gemm_gather_tc`` / ``xb_wgrad_gather_tc``, include/xb200.h): geometry builders that express the
NatureCNN layers (xuance/torch/rl_models/representations/cnn.py:45-50, 84-101; modules/layers.py:16-65), their data
gradients and weight gradients as the gathered-operand GEMM of ``xuance_b200/csrc/conv_index.h``, thin launch wrappers, and
``TensorCoreNatureCNN`` - the forward / backward orchestration behind ``compute="tc"`` of the pixel encoders.

The geometry and the kernel's index arithmetic are verified on the host (tests/test_conv_index.py emulates the
shared-memory staging, the descriptor reads and the per-plane MMA issue and compares with ``torch.nn.functional.conv2d`` /
autograd); tests/test_gpu_tc_conv.py pins every mode against float64 on the GPU.
"""
from dataclasses import dataclass, field
from typing import List

import numpy as np
import torch

from ... import _lib

KC = 64          # XB_CONV_KC
MAX_TAPS = 64    # XB_CONV_MAX_TAPS


@dataclass
class GatherGeometry:
    """One ``xb_gemm_gather_tc`` call: sites [B, OY, OX] over an NHWC input [B, IH, IW, C]; tap t reads
    (y*sy + dy[t], x*sx + dx[t]); the site's result row lands at (y*oys + oy0, x*oxs + ox0) of a [B, out_H, out_W] grid.
    ``fold`` > 1: ``fold`` horizontally adjacent pixels were folded into the channel axis (input viewed as
    [B, IH, W/fold, C*fold]) so that every 16-byte unit is 8 contiguous bf16 values."""
    B: int
    IH: int
    IW: int
    C: int
    OY: int
    OX: int
    sy: int
    sx: int
    dy: List[int]
    dx: List[int]
    out_H: int
    out_W: int
    oys: int = 1
    oxs: int = 1
    oy0: int = 0
    ox0: int = 0
    fold: int = 1
    taps: List[tuple] = field(default_factory=list)    # (kh, kw) of the ORIGINAL kernel per tap (before folding)

    @property
    def T(self):
        return len(self.dy)

    @property
    def K(self):
        return self.T * self.C

    @property
    def M(self):
        return self.B * self.OY * self.OX

    def check(self):
        assert self.C % 8 == 0, "channels per tap must be a multiple of 8 (one 16-byte unit)"
        assert self.K % KC == 0, "K = taps*channels must be a multiple of %d" % KC
        assert self.T <= MAX_TAPS
        assert all(-128 <= v <= 127 for v in self.dy + self.dx)
        assert (self.OY - 1) * self.oys + self.oy0 < self.out_H and (self.OX - 1) * self.oxs + self.ox0 < self.out_W
        return self


def conv_out(size, k, stride, pad):
    return (size + 2 * pad - k) // stride + 1


def conv_forward_geometry(B, H, W, C, KH, KW, stride, pad):
    """y = conv2d(x, w, stride, pad) with x NHWC [B,H,W,C] and the weight packed as [N, (kh, kw, c)]."""
    OY, OX = conv_out(H, KH, stride, pad), conv_out(W, KW, stride, pad)
    fold = 1
    if C % 8 != 0:
        assert 8 % C == 0, "channel counts below 8 must divide 8"
        fold = 8 // C
        assert W % fold == 0 and KW % fold == 0 and stride % fold == 0 and pad % fold == 0, \
            "folding %d pixels into the channel axis needs W, KW, stride and pad divisible by %d" % (fold, fold)
    dy, dx, taps = [], [], []
    for kh in range(KH):
        for kw2 in range(KW // fold):
            dy.append(kh - pad)
            dx.append(kw2 - pad // fold)
            taps.append((kh, kw2 * fold))
    return GatherGeometry(B=B, IH=H, IW=W // fold, C=C * fold, OY=OY, OX=OX, sy=stride, sx=stride // fold, dy=dy, dx=dx,
                          out_H=OY, out_W=OX, fold=fold, taps=taps).check()


def linear_geometry(B, in_features):
    """y = x @ W^T : one tap, one site per row."""
    return GatherGeometry(B=B, IH=1, IW=1, C=in_features, OY=1, OX=1, sy=1, sx=1, dy=[0], dx=[0], out_H=1, out_W=1,
                          taps=[(0, 0)]).check()


def conv_dgrad_geometries(B, H, W, C, KH, KW, stride, pad, N):
    """dx = conv2d_backward_input(dy): one GEMM per stride phase (iy % s, ix % s) over the output gradient
    dy NHWC [B, OY, OX, N]; each phase uses the kernel taps with kh = (py + pad) mod s, and writes the input-gradient
    pixels of its phase.  Returns [(geometry, [(kh, kw), ...])]; the matching weight matrix of a phase is
    [C, (tap, n)] = w[n, c, kh, kw]."""
    OY, OX = conv_out(H, KH, stride, pad), conv_out(W, KW, stride, pad)
    out = []
    for py in range(stride):
        for px in range(stride):
            ny, nx = (H - py + stride - 1) // stride, (W - px + stride - 1) // stride
            if ny <= 0 or nx <= 0:
                continue
            dy, dx, taps = [], [], []
            for kh in range(KH):
                if (py + pad - kh) % stride:
                    continue
                for kw in range(KW):
                    if (px + pad - kw) % stride:
                        continue
                    dy.append((py + pad - kh) // stride)
                    dx.append((px + pad - kw) // stride)
                    taps.append((kh, kw))
            if not taps:
                continue
            g = GatherGeometry(B=B, IH=OY, IW=OX, C=N, OY=ny, OX=nx, sy=1, sx=1, dy=dy, dx=dx, out_H=H, out_W=W,
                               oys=stride, oxs=stride, oy0=py, ox0=px, taps=taps).check()
            out.append((g, taps))
    return out


def dgrad_weight_matrix(w, taps):
    """torch conv weight [N, C, KH, KW] -> [C, (tap, n)] float32 for the taps of one dgrad phase."""
    cols = [w[:, :, kh, kw].t() for kh, kw in taps]          # each [C, N]
    return torch.cat(cols, dim=1).contiguous()


# ------------------------------------------------------------------------------------------------ device wrappers
# Operands are "plane tensors": bfloat16 [P, ...] with x = planes.sum(0); plane q = bf16 of the residual the planes before
# it leave.  P = 1 is exact for raw uint8 pixels (integers <= 256), P = 2 is exact to 2^-16, P = 3 to 2^-24.  A K12 launch
# multiplies an A operand of PA planes with a B operand of PB >= PA planes and keeps the products whose plane indices sum
# to < PB, each order of magnitude in its own float32 accumulator (added smallest first in the epilogue - the tensor core
# truncates when it adds into an accumulator, DESIGN.md section 4).
def split_bf16(x, planes=2):
    """float32 CUDA tensor -> bfloat16 [planes, *x.shape]."""
    x = x.contiguous()
    out = torch.empty((planes,) + tuple(x.shape), dtype=torch.bfloat16, device=x.device)
    _lib.call("xb_split_bf16", _lib.ptr(x), x.numel(), planes, _lib.ptr(out))
    return out


def pack_weights(jobs, planes, device):
    """Several operand forms in ONE launch (``xb_pack_weights``).  ``jobs``: list of (w [N, C, KH, KW] float32, mode, taps, scale)
    with mode _lib.PACK_FORWARD -> [planes, N, KH*KW*C], PACK_TRANSPOSED -> [planes, KH*KW*C, N], PACK_DGRAD -> [planes, C,
    len(taps)*N] (taps = [(kh, kw), ...]); returns the bfloat16 plane tensors in job order."""
    import ctypes
    arr = (_lib.XbPackJob * len(jobs))()
    outs = []
    for j, (w, mode, taps, scale) in enumerate(jobs):
        assert w.is_contiguous() and w.dtype == torch.float32 and w.dim() == 4
        N, C, KH, KW = w.shape
        shape = {_lib.PACK_FORWARD: (N, KH * KW * C), _lib.PACK_TRANSPOSED: (KH * KW * C, N),
                 _lib.PACK_DGRAD: (C, len(taps or ()) * N)}[mode]
        out = torch.empty((planes,) + shape, dtype=torch.bfloat16, device=device)
        J = arr[j]
        J.w, J.out, J.N, J.C, J.KH, J.KW, J.mode, J.scale, J.planes = w.data_ptr(), out.data_ptr(), N, C, KH, KW, mode, scale, planes
        J.n_taps = len(taps) if mode == _lib.PACK_DGRAD else 0
        for t, (kh, kw) in enumerate(taps or ()):
            J.kh[t], J.kw[t] = kh, kw
        outs.append(out)
    _lib.call("xb_pack_weights", ctypes.addressof(arr), len(jobs))
    return outs


def pack_conv_weight(w, planes=2, scale=1.0):
    """[N, C, KH, KW] float32 CUDA -> bfloat16 [planes, N, KH*KW*C] in (kh, kw, c) column order, times ``scale``."""
    w = w.contiguous()
    N, C, KH, KW = w.shape
    out = torch.empty((planes, N, KH * KW * C), dtype=torch.bfloat16, device=w.device)
    _lib.call("xb_pack_conv_weight", _lib.ptr(w), N, C, KH, KW, planes, float(scale), _lib.ptr(out))
    return out


def n_tile_for(N, planes_b):
    """Columns per work item: the largest multiple of 32 that divides N with planes_b * n_tile <= 256 (the register
    accumulators of a consumer thread hold planes_b * n_tile / 2 floats)."""
    t = (256 // planes_b) // 32 * 32
    while t >= 32:
        if N % t == 0:
            return t
        t -= 32
    raise ValueError("N = %d has no column tile that is a multiple of 32" % N)


def _plane_arg(t):
    """(pointer of plane 0, plane stride in elements) of a plane tensor whose planes are each contiguous."""
    assert t[0].is_contiguous(), "each plane must be contiguous"
    return _lib.ptr(t[0]), t.stride(0)


_TAPS = {}
flop_log = None      # bench.py: when a list, every K12 launch appends (abi name, layer tag, executed bf16 FLOPs, fp32-equivalent FLOPs)


def _products(pa, pb):
    """Plane products one launch executes: A plane i meets the first pb - i B planes."""
    return sum(pb - i for i in range(pa))


def _log_flops(name, rows, cols, depth, pa, pb, useful=None):
    """bench.py's roofline log: the ALGORITHMIC flops of a launch - 2 * useful * depth with ``useful`` = (rows x cols) pairs
    that are real outputs (padding / halo / garbage sites of the padded layouts excluded; default rows * cols) - times the
    plane products float32-grade arithmetic needs, and the same without the plane factor (float32-equivalent)."""
    if flop_log is not None:
        eq = 2.0 * (rows * cols if useful is None else useful) * depth
        flop_log.append((name, "M=%d N=%d K=%d PA=%d PB=%d" % (rows, cols, depth, pa, pb), eq * _products(pa, pb), eq))


def _taps(geom):
    """int8 host arrays of the tap offsets (kept alive per geometry: the ABI copies them at launch time)."""
    key = (tuple(geom.dy), tuple(geom.dx))
    if key not in _TAPS:
        _TAPS[key] = (torch.tensor(geom.dy, dtype=torch.int8), torch.tensor(geom.dx, dtype=torch.int8))
    return _TAPS[key]


def gemm_gather(x_pl, w_pl, geom, bias=None, relu=False, out_f32=None, out_pl=None, out_ld=None, out_c0=0, relu_mask=None,
                n_tile=None, mask_ld=0, mask_c0=0, colsum=None):
    """One K12 launch.  ``x_pl`` [PA, B, IH, IW, C] (any shape with that element order), ``w_pl`` [PB, N, K]; outputs are
    caller-allocated: ``out_f32`` [rows, out_ld] and / or ``out_pl`` [P_out, rows, out_ld]; ``colsum`` float32
    [ceil(M / 128), N] receives the per-tile column sums of the result (bias-gradient partials, see ``bias_grad``)."""
    PB, N, K = w_pl.shape
    PA = x_pl.shape[0]
    assert K == geom.K and PA <= PB, (K, geom.K, PA, PB)
    out_ld = N if out_ld is None else out_ld
    n_tile = n_tile_for(N, PB) if n_tile is None else n_tile
    dy, dx = _taps(geom)
    xp, xs = _plane_arg(x_pl)
    wp, ws = _plane_arg(w_pl)
    op, os_ = _plane_arg(out_pl) if out_pl is not None else (None, 0)
    _log_flops("xb_gemm_gather_tc", geom.M, N, K, PA, PB)
    _lib.call("xb_gemm_gather_tc", PA, PB, xp, xs, wp, ws, _lib.ptr(bias) if bias is not None else None,
              _lib.ptr(relu_mask) if relu_mask is not None else None, mask_ld, mask_c0, geom.B, geom.IH, geom.IW, geom.C,
              geom.OY, geom.OX,
              geom.sy, geom.sx, geom.T, dy.data_ptr(), dx.data_ptr(), N, n_tile, 1 if relu else 0, op, os_,
              out_pl.shape[0] if out_pl is not None else 0, _lib.ptr(out_f32) if out_f32 is not None else None, geom.out_H,
              geom.out_W, geom.oys, geom.oxs, geom.oy0, geom.ox0, out_ld, out_c0, _lib.ptr(colsum) if colsum is not None else None)
    return out_f32, out_pl


def bias_grad(colsum, N, out=None, accumulate=False):
    """Column-sum partials (any shape [..., N], contiguous) -> [N]: the bias gradient of the layer whose output gradient the
    producing K12 launch wrote; the partials are added in a fixed order by xb_wgrad_reduce (which uses them as scratch)."""
    return wgrad_reduce(colsum.view(-1, 1, N), N, 1, 1, 1, out=out, accumulate=accumulate).view(N)


def wgrad_gather(x_pl, g_pl, geom, splits, n_tile=None):
    """Partial weight gradients [splits, K, N] (float32) of the gathered GEMM ``geom`` for the output gradient planes
    ``g_pl`` [PB, sites, N]."""
    PB, _, N = g_pl.shape
    PA = x_pl.shape[0]
    assert PA <= PB and g_pl.stride(2) == 1
    n_tile = n_tile_for(N, PB) if n_tile is None else n_tile
    partials = torch.empty((splits, geom.K, N), dtype=torch.float32, device=g_pl.device)
    dy, dx = _taps(geom)
    xp, xs = _plane_arg(x_pl)
    um = getattr(geom, "useful_M", None)
    _log_flops("xb_wgrad_gather_tc", geom.K, N, geom.M, PA, PB, useful=None if um is None else geom.K * N * um / geom.M)
    _lib.call("xb_wgrad_gather_tc", PA, PB, xp, xs, _lib.ptr(g_pl), g_pl.stride(0), g_pl.stride(1), geom.B, geom.IH, geom.IW,
              geom.C, geom.OY, geom.OX, geom.sy, geom.sx, geom.T, dy.data_ptr(), dx.data_ptr(), N, n_tile, splits,
              _lib.ptr(partials))
    return partials


def wgrad_reduce(partials, N, C, KH, KW, out=None, accumulate=False, scale=1.0):
    """[splits, (kh,kw,c), N] partials -> torch-layout weight gradient [N, C, KH, KW] (times ``scale``)."""
    out = torch.empty((N, C, KH, KW), dtype=torch.float32, device=partials.device) if out is None else out
    _lib.call("xb_wgrad_reduce", _lib.ptr(partials), partials.shape[0], N, C, KH, KW, float(scale), _lib.ptr(out),
              1 if accumulate else 0)
    return out


def wgrad_splits(M, K, n_tiles=1, sm_count=132):
    """Split count for the weight gradient: about two work items per SM, at least 8 chunks of 64 sites per split, at most
    4096 sites per split (the tensor core truncates on every addition into the accumulator: a chain of n K-steps carries a
    bias of up to n * 2^-24 relative, so long reductions are cut and the pieces added in float32 by xb_wgrad_reduce), and
    the rule of ``xb_wgrad_sites_per_split`` (no empty split)."""
    m_tiles = -(-K // 128) * n_tiles
    s = max(1, min((2 * sm_count) // m_tiles, M // (8 * KC)))
    s = max(s, -(-M // 4096))
    while s > 1:
        per = -(-(-(-M // s)) // KC) * KC
        if (s - 1) * per < M:
            break
        s -= 1
    return s


class CudaBackend:
    """The product backend of ``TensorCoreNatureCNN``: every method is one or a few C-ABI launches (K12).  The host test
    substitutes an emulated backend with the same methods (tests/test_conv_index.py) to check the orchestration."""

    def __init__(self, planes=3):
        self.planes = planes

    def split(self, x):
        return split_bf16(x, self.planes)

    def pack_weight(self, w4d, scale=1.0):
        return pack_conv_weight(w4d, self.planes, scale)

    def empty_planes(self, shape, like):
        return torch.empty((self.planes,) + tuple(shape), dtype=torch.bfloat16, device=like.device)

    def empty_f32(self, shape, like):
        return torch.empty(shape, dtype=torch.float32, device=like.device)

    def gemm(self, x_pl, w_pl, geom, bias=None, relu=False, out_f32=None, out_pl=None, out_ld=None, out_c0=0, mask=None):
        gemm_gather(x_pl, w_pl, geom, bias=bias, relu=relu, out_f32=out_f32, out_pl=out_pl, out_ld=out_ld, out_c0=out_c0,
                    relu_mask=mask)

    def wgrad(self, x_pl, g_pl, geom, N, C, KH, KW, scale=1.0, out=None, accumulate=False):
        nt = N // n_tile_for(N, g_pl.shape[0])
        splits = wgrad_splits(geom.M, geom.K, nt)
        return wgrad_reduce(wgrad_gather(x_pl, g_pl, geom, splits), N, C, KH, KW, scale=scale, out=out, accumulate=accumulate)

    def colsum(self, g_pl):
        # bias gradient: reduce the bf16 planes straight into float32 (no float32 copy of the [P, sites, N] tensor)
        return g_pl.sum(dim=1, dtype=torch.float32).sum(0)

    def to_float(self, pl):
        return pl.float().sum(0)


class TensorCoreNatureCNN:
    """The convolution stack + hidden layer of AC_CNN_Atari / Basic_CNN's conv part (cnn.py:45-50, 84-101) as K12 launches,
    forward AND backward, for one batch size.  Activations live as bf16 plane tensors (NHWC) between layers; the ReLU
    derivative is applied inside the data-gradient GEMM's epilogue from plane 0 of the saved activation.

    The input is either ``planes`` planes of the normalised observation x/255, or ONE plane holding the raw uint8 pixel
    values (exact in bf16): then the first layer's packed weights and its weight gradient carry the 1/255, the layer's A
    operand costs a third of the traffic and a third of the tensor work, and the minibatch gather writes one plane.

    ``convs``: nn.Conv2d modules (padding (k - s)//2 as layers.py:46 builds them), each followed by ReLU;
    ``fc``: nn.Linear over the NCHW-flattened last feature map, followed by ReLU."""

    def __init__(self, convs, fc, in_hwc, backend=None):
        self.convs, self.fc = list(convs), fc
        self.in_hwc = tuple(in_hwc)
        self.be = backend if backend is not None else CudaBackend()
        self._plans = {}

    def parameters(self):
        ps = []
        for c in self.convs:
            ps += [c.weight, c.bias]
        if self.fc is not None:
            ps += [self.fc.weight, self.fc.bias]
        return ps

    def _plan(self, B):
        if B in self._plans:
            return self._plans[B]
        H, W, C = self.in_hwc
        layers = []
        for conv in self.convs:
            N, Cw, KH, KW = conv.weight.shape
            s, p = conv.stride[0], conv.padding[0]
            assert Cw == C and conv.stride[0] == conv.stride[1] and conv.padding[0] == conv.padding[1]
            fwd = conv_forward_geometry(B, H, W, C, KH, KW, s, p)
            dgrad = conv_dgrad_geometries(B, H, W, C, KH, KW, s, p, N) if layers else None   # no gradient w.r.t. pixels
            layers.append(dict(kind="conv", N=N, C=C, KH=KH, KW=KW, fwd=fwd, dgrad=dgrad))
            H, W, C = fwd.OY, fwd.OX, N
        if self.fc is not None:
            N, K = self.fc.weight.shape
            assert K == H * W * C
            layers.append(dict(kind="fc", N=N, C=C, KH=H, KW=W, fwd=linear_geometry(B, K), dgrad=linear_geometry(B, N)))
        self._plans[B] = layers
        return layers

    # ---- forward: returns float32 [sites of the last layer, features]; keeps what backward needs
    def forward(self, x_pl, B, keep=True):
        """``keep=False`` (inference under no_grad): nothing a pending backward needs is overwritten."""
        be, plan = self.be, self._plan(B)
        raw = x_pl.shape[0] == 1 and be.planes > 1          # one exact plane of uint8 values: 1/255 goes into the weights
        saved, cur, out_f32 = [], x_pl, None
        for li, L in enumerate(plan):
            mod = self.convs[li] if L["kind"] == "conv" else self.fc
            N, g = L["N"], L["fwd"]
            w4 = (mod.weight if L["kind"] == "conv" else mod.weight.reshape(N, L["C"], L["KH"], L["KW"])).detach()
            scale = 1.0 / 255.0 if (raw and li == 0) else 1.0
            w_pl = be.pack_weight(w4, scale)
            out_pl = be.empty_planes((g.M, N), cur)
            out_f32 = be.empty_f32((g.M, N), cur) if li == len(plan) - 1 else None
            be.gemm(cur, w_pl, g, bias=mod.bias.detach(), relu=True, out_f32=out_f32, out_pl=out_pl, out_ld=N)
            saved.append(dict(x=cur, y=out_pl, w4=w4, scale=scale))
            cur = out_pl
        if keep:
            self._saved = (B, saved)
        return out_f32

    # ---- backward: dz float32 = gradient w.r.t. the array forward() returned; returns gradients in parameters() order
    def backward(self, dz):
        be = self.be
        B, saved = self._saved
        plan = self._plan(B)
        grads = [None] * (2 * len(plan))
        y_last = saved[-1]["y"]
        g_pl = be.split(dz * (y_last[0] > 0).to(dz.dtype))            # ReLU derivative of the last layer (plane 0 > 0)
        for li in range(len(plan) - 1, -1, -1):
            L, sv = plan[li], saved[li]
            N, C, KH, KW = L["N"], L["C"], L["KH"], L["KW"]
            # -- weight and bias gradients (the weight gradient gathers exactly like the forward)
            dw = be.wgrad(sv["x"], g_pl, L["fwd"], N, C, KH, KW, sv["scale"])
            grads[2 * li] = dw if L["kind"] == "conv" else dw.reshape(N, C * KH * KW)
            grads[2 * li + 1] = be.colsum(g_pl)
            if li == 0:
                break
            # -- data gradient, masked by the previous activation's ReLU derivative inside the GEMM epilogue
            prev_y = saved[li - 1]["y"]                   # [P, sites_prev, C] == NHWC input planes of this layer
            out_pl = be.empty_planes(tuple(prev_y.shape[1:]), prev_y)
            if L["kind"] == "conv":
                for geom, taps in L["dgrad"]:
                    w_pl = be.split(dgrad_weight_matrix(sv["w4"], taps))          # [P, C, (tap, n)]
                    be.gemm(g_pl, w_pl, geom, out_pl=out_pl, out_ld=C, mask=prev_y[0])
            else:
                K = C * KH * KW
                w_pl = be.split(sv["w4"].permute(0, 2, 3, 1).reshape(N, K).t().contiguous())   # [P, K (h,w,c), N]
                be.gemm(g_pl, w_pl, L["dgrad"], out_pl=out_pl, out_ld=K, mask=prev_y[0])
            g_pl = out_pl
        return grads


# ------------------------------------------------------------------------------------------------ padded-row layouts + TMA boxes
@dataclass
class BoxGeometry:
    """One ``xb_gemm_box_tc`` call (include/xb200.h): a convolution over an activation stored with padded rows
    [planes][B*hp_in][W][C]; see ConvParams.a_box in conv_tc.cu."""
    B: int
    C: int
    W: int
    hp_in: int
    box_c: int
    box_px: int
    box_h: int
    row_step: int
    chunks: List[tuple]          # (c0, w0, r0) per 64-deep K chunk
    hp_out: int
    y0: int
    y1: int
    out_H: int
    out_W: int
    oys: int = 1
    oxs: int = 1
    oy0: int = 0
    ox0: int = 0
    mask_W: int = 0              # ReLU mask tensor: pixels per row / pixel offset when it is not laid out like the output
    mask_x0: int = 0

    @property
    def sites_per_row(self):
        return self.box_px

    @property
    def K(self):
        return 64 * len(self.chunks)

    @property
    def M(self):                  # rows the kernel computes (padded grid)
        return self.B * self.hp_out * self.sites_per_row

    @property
    def m_tiles(self):            # work items along M (rows of a ``colsum`` buffer)
        return -(-self.B * self.hp_out // self.box_h)


_BOXTAB = {}
import os as _os
# weight gradients with both operands as TMA boxes, per layer (measured at B = 8192, 3 planes: conv3 785 us box vs 837 us
# gathered; conv2 947 us box vs 851 us gathered - its 16 pixel-pair chunks re-read G once per pair of chunks)
BOX_WGRAD = _os.environ.get("XB_K12_BOX_WGRAD", "3")
BOX_WGRAD2, BOX_WGRAD3 = "2" in BOX_WGRAD, "3" in BOX_WGRAD
# xb_gemm_halo_tc (activation tile resident in shared memory, taps = descriptor offsets): "2" = conv2's data gradient (its
# four stride phases become ONE launch: 868 us vs 892 us as four box launches at B = 8192), "3" = also conv3 forward / data
# gradient (473 / 479 us vs 461 / 469 us as box launches: no gain - with 64-column tiles the tensor pipe waits for its own
# shared-memory operand reads, not for the fill of the ring, see DESIGN.md section 3a), "0" = box launches only
HALO_MODE = _os.environ.get("XB_K12_HALO", "2")
HALO, HALO3 = HALO_MODE != "0", HALO_MODE in ("1", "3")


def gemm_box(x_pl, w_pl, bg, bias=None, relu=False, out_f32=None, out_pl=None, out_ld=None, out_c0=0, relu_mask=None,
             n_tile=None, colsum=None):
    """One K12 launch with the A operand fetched by TMA boxes (``x_pl`` [PA, B*hp_in, W, C], padded rows)."""
    PB, N, K = w_pl.shape
    PA = x_pl.shape[0]
    assert K == bg.K and PA <= PB and tuple(x_pl.shape[1:]) == (bg.B * bg.hp_in, bg.W, bg.C), (x_pl.shape, bg)
    out_ld = N if out_ld is None else out_ld
    n_tile = n_tile_for(N, PB) if n_tile is None else n_tile
    key = tuple(bg.chunks)
    if key not in _BOXTAB:
        _BOXTAB[key] = tuple(torch.tensor([c[i] for c in bg.chunks], dtype=torch.int16) for i in range(3))
    c0, w0, r0 = _BOXTAB[key]
    xp, xs = _plane_arg(x_pl)
    wp, ws = _plane_arg(w_pl)
    op, os_ = _plane_arg(out_pl) if out_pl is not None else (None, 0)
    _log_flops("xb_gemm_box_tc", bg.M, N, K, PA, PB, useful=bg.B * (bg.y1 - bg.y0 + 1) * bg.box_px * N)
    _lib.call("xb_gemm_box_tc", PA, PB, xp, xs, bg.C, bg.W, bg.B * bg.hp_in, bg.box_c, bg.box_px, bg.box_h, bg.row_step,
              len(bg.chunks), c0.data_ptr(), w0.data_ptr(), r0.data_ptr(), wp, ws,
              _lib.ptr(bias) if bias is not None else None, _lib.ptr(relu_mask) if relu_mask is not None else None,
              bg.mask_W, bg.mask_x0, bg.B, bg.hp_out, bg.y0, bg.y1, N, n_tile, 1 if relu else 0, op, os_,
              out_pl.shape[0] if out_pl is not None else 0, _lib.ptr(out_f32) if out_f32 is not None else None,
              bg.out_H, bg.out_W, bg.oys, bg.oxs, bg.oy0, bg.ox0, out_ld, out_c0, _lib.ptr(colsum) if colsum is not None else None)


@dataclass
class HaloGeometry:
    """One ``xb_gemm_halo_tc`` call (include/xb200.h): stride-1 gathers over a 64-channel padded-row tensor
    [planes][B*hp][W][64] with the activation tile resident in shared memory; ``subs`` = one entry per sub-item
    (n tile / stride phase): dict(shifts=[(dr, dc), ...], y1, x1, oy0, ox0)."""
    B: int
    W: int
    hp: int
    halo_w: int
    halo_w0: int
    subs: List[dict]
    y0: int
    N: int
    out_H: int
    out_W: int
    oys: int = 1
    oxs: int = 1
    same_cols: bool = False
    mask_W: int = 0
    mask_x0: int = 0

    @property
    def n_chunks(self):
        return len(self.subs[0]["shifts"])

    @property
    def K(self):
        return 64 * self.n_chunks

    @property
    def M(self):                  # positions of the haloed raster (rows the kernel computes)
        return self.B * self.hp * self.halo_w

    @property
    def m_tiles(self):            # work items along M times sub-items (rows of a ``colsum`` buffer)
        return -(-self.M // 128) * len(self.subs)


_HALOTAB = {}


def gemm_halo(x_pl, w_pl, hg, bias=None, relu=False, out_f32=None, out_pl=None, out_ld=None, out_c0=0, relu_mask=None, colsum=None):
    """One K12 launch in halo mode (``x_pl`` [PA, B*hp, W, 64] padded rows, ``w_pl`` [PB, n_sub*N, n_chunks*64])."""
    PB, Nw, K = w_pl.shape
    PA = x_pl.shape[0]
    n_sub = len(hg.subs)
    assert K == hg.K and Nw == n_sub * hg.N and PA <= PB and tuple(x_pl.shape[1:]) == (hg.B * hg.hp, hg.W, 64), (x_pl.shape, w_pl.shape)
    out_ld = (hg.N if hg.same_cols else Nw) if out_ld is None else out_ld
    key = id(hg)
    if key not in _HALOTAB:
        i16 = lambda v: torch.tensor(v, dtype=torch.int16)
        _HALOTAB[key] = (hg, i16([d[0] for sb in hg.subs for d in sb["shifts"]]), i16([d[1] for sb in hg.subs for d in sb["shifts"]]),
                         i16([sb["y1"] for sb in hg.subs]), i16([sb["x1"] for sb in hg.subs]),
                         i16([sb["oy0"] for sb in hg.subs]), i16([sb["ox0"] for sb in hg.subs]))
    _, dr, dc, y1, x1, oy0, ox0 = _HALOTAB[key]
    xp, xs = _plane_arg(x_pl)
    wp, ws = _plane_arg(w_pl)
    op, os_ = _plane_arg(out_pl) if out_pl is not None else (None, 0)
    _log_flops("xb_gemm_halo_tc", hg.M, Nw, K, PA, PB, useful=sum(hg.B * (sb["y1"] - hg.y0 + 1) * (sb["x1"] + 1) * hg.N for sb in hg.subs))
    _lib.call("xb_gemm_halo_tc", PA, PB, xp, xs, hg.W, hg.B * hg.hp, hg.halo_w, hg.halo_w0, n_sub, hg.n_chunks, dr.data_ptr(),
              dc.data_ptr(), wp, ws, _lib.ptr(bias) if bias is not None else None,
              _lib.ptr(relu_mask) if relu_mask is not None else None, hg.mask_W, hg.mask_x0, hg.B, hg.hp, hg.y0, y1.data_ptr(),
              x1.data_ptr(), hg.N, 1 if relu else 0, op, os_, out_pl.shape[0] if out_pl is not None else 0,
              _lib.ptr(out_f32) if out_f32 is not None else None, hg.out_H, hg.out_W, hg.oys, hg.oxs, oy0.data_ptr(), ox0.data_ptr(),
              out_ld, out_c0, 1 if hg.same_cols else 0, _lib.ptr(colsum) if colsum is not None else None)


def wgrad_box(x_pl, g_pl, bg, box_h, splits):
    """Partial weight gradients [splits, K, N] of the convolution ``bg`` (its forward BoxGeometry) with both operands fetched
    by TMA boxes: ``x_pl`` [PA, B*hp_in, W, C] padded input, ``g_pl`` [PB, B*hp_out, sites_per_row, N] padded output gradient;
    a reduction chunk is ``box_h`` grid rows."""
    PB, g_rows, spr, N = g_pl.shape
    PA = x_pl.shape[0]
    assert spr == bg.sites_per_row and g_rows == bg.B * bg.hp_out and PA <= PB
    key = tuple(bg.chunks)
    if key not in _BOXTAB:
        _BOXTAB[key] = tuple(torch.tensor([c[i] for c in bg.chunks], dtype=torch.int16) for i in range(3))
    c0, w0, r0 = _BOXTAB[key]
    partials = torch.empty((splits, bg.K, N), dtype=torch.float32, device=g_pl.device)
    xp, xs = _plane_arg(x_pl)
    _log_flops("xb_wgrad_box_tc", bg.K, N, g_rows * spr, PA, PB, useful=bg.K * N * (bg.B * (bg.y1 - bg.y0 + 1) * spr) / (g_rows * spr))
    _lib.call("xb_wgrad_box_tc", PA, PB, xp, xs, bg.C, bg.W, bg.B * bg.hp_in, bg.box_c, bg.box_px, box_h, bg.row_step,
              len(bg.chunks), c0.data_ptr(), w0.data_ptr(), r0.data_ptr(), _lib.ptr(g_pl), g_pl.stride(0), g_rows, N, splits,
              _lib.ptr(partials))
    return partials


def wgrad_box_splits(g_rows, box_h, K, N, sm_count=132):
    """Splits for the box weight gradient: about two work items per SM, chains of at most 4096 sites (truncating adds)."""
    tiles = -(-K // 128) * (N // 64)
    s = max(1, (2 * sm_count) // tiles, -(-g_rows * 10 // 4096))
    s = min(s, max(1, g_rows // (4 * box_h)))
    while s > 1:
        per = -(-(-(-g_rows // s)) // box_h) * box_h
        if (s - 1) * per < g_rows:
            break
        s -= 1
    return s


class BoxNatureCNN(TensorCoreNatureCNN):
    """``TensorCoreNatureCNN`` with the activations between the convolutions kept in PADDED-ROW layouts so that the A
    operands of every convolution after the first (forward and data gradient) are plain TMA boxes instead of 16-byte
    cp.async gathers - a CTA's cp.async stream is limited by L1 miss tracking, well below what the
    tensor pipe needs for these 64-column layers.

    Layout of an activation with H real rows: [P, B, hp, W, C], real row i at row i + off, every other row zero (written once
    at allocation and never again).  A layer with stride s reads input row s*y' + r0[kh] for its output (padded) row y', which
    requires hp_in = s * hp_out; garbage rows of the padded output grid are computed and dropped.  A TMA box must have a
    128-byte inner extent (measured with tools/tma_probe.py: a 64-byte inner box under the 128-byte swizzle still takes one
    128-byte shared-memory row per pixel), so the 32-channel activation of the first convolution is stored W1p = W1 + 1
    pixels wide with ONE zero pixel on the left and read as 64-channel PIXEL PAIRS: the taps (kh, kw0), (kh, kw0 + 1) of the
    stride-2 convolution are pair x + kw0 / 2 for output pixel x.  Supported after the first convolution: (C_in = 32, s = 2,
    odd padding, even kernel) and (C_in = 64, s = 1) - the NatureCNN / Basic_CNN stacks; the first convolution (raw uint8
    plane, 4 channels) and its weight gradient keep the gathered path, with the padded tensors described to it as ordinary
    geometries."""

    grads_ready = None      # optional callable(first_final_parameter), see backward()

    def _box_ok(self):
        cs = self.convs
        if len(cs) != 3:
            return False
        c1, c2, c3 = cs
        return (c2.in_channels == 32 and c2.stride[0] == 2 and c2.kernel_size[0] % 2 == 0 and c2.padding[0] % 2 == 1
                and c3.in_channels == 64
                and c3.stride[0] == 1 and c2.out_channels == 64 and c3.out_channels == 64 and c1.out_channels == 32)

    def _plan(self, B):
        if B in self._plans:
            return self._plans[B]
        assert self._box_ok(), "BoxNatureCNN: unsupported convolution stack"
        H, W, C = self.in_hwc
        c1, c2, c3 = self.convs
        k1, s1, p1 = c1.kernel_size[0], c1.stride[0], c1.padding[0]
        k2, s2, p2 = c2.kernel_size[0], c2.stride[0], c2.padding[0]
        k3, s3, p3 = c3.kernel_size[0], c3.stride[0], c3.padding[0]
        H1, W1 = conv_out(H, k1, s1, p1), conv_out(W, k1, s1, p1)          # 21 x 21
        H2, W2 = conv_out(H1, k2, s2, p2), conv_out(W1, k2, s2, p2)        # 10 x 10
        H3, W3 = conv_out(H2, k3, s3, p3), conv_out(W2, k3, s3, p3)        # 10 x 10
        assert H3 == H2 and W3 == W2 and W2 * 2 <= 256
        # padded grids: conv3's sites and conv2's sites share hp2 rows per image (valid rows 1 .. H2); conv2 reads act1 with
        # row step 2, so act1 has hp1 = 2 * hp2 rows per image
        hp2 = H2 + 2
        hp1 = 2 * hp2
        off1 = p2 + 2 * 1                                                    # real row i of act1 at padded row i + off1
        assert off1 + H1 <= hp1
        # act1 pixel i at column i + xo1 of W1p (even) columns: column 2x + kw0 - p2 + xo1 of tap kw0 (even) is even
        xo1 = p2 % 2
        W1p = -(-max(W1 + xo1, 2 * (W2 - 1) + k2 - p2 + xo1) // 2) * 2
        P = dict(B=B, H=H, W=W, C=C, H1=H1, W1=W1, H2=H2, W2=W2, hp1=hp1, hp2=hp2, off1=off1, W1p=W1p, xo1=xo1,
                 N1=c1.out_channels, N2=c2.out_channels, N3=c3.out_channels)
        # ---- conv1 forward (gathered, raw plane) writing into act1's padded layout
        g1 = conv_forward_geometry(B, H, W, C, k1, k1, s1, p1)
        g1.out_H, g1.oy0 = hp1, off1
        g1.out_W, g1.ox0 = W1p, xo1
        P["fwd1"] = g1
        # conv1 weight gradient: the sites are ALL rows of the padded act1 grid (zero gradient rows contribute nothing)
        w1 = conv_forward_geometry(B, H, W, C, k1, k1, s1, p1)
        w1.OY = hp1
        w1.dy = [d - s1 * off1 for d in w1.dy]
        w1.out_H = hp1
        P["wg1"] = w1.check()
        P["wg1"].useful_M = B * H1 * W1
        # ---- conv2 forward (box over act1's pixel-pair view [B*hp1, W1p/2, 64]): chunk = (kh, kw0 and kw0 + 1) x 32 channels
        ch2 = [(0, (kw - p2 + xo1) // 2, kh) for kh in range(k2) for kw in range(0, k2, 2)]
        P["fwd2"] = BoxGeometry(B=B, C=64, W=W1p // 2, hp_in=hp1, box_c=64, box_px=W2, box_h=hp2, row_step=2, chunks=ch2,
                                hp_out=hp2, y0=1, y1=H2, out_H=hp2, out_W=W2, oy0=1)
        P["wg2"] = GatherGeometry(B=B, IH=hp1, IW=W1p, C=32, OY=hp2, OX=W2, sy=2, sx=2,
                                  dy=[kh for kh in range(k2) for _ in range(k2)],
                                  dx=[kw - p2 + xo1 for _ in range(k2) for kw in range(k2)], out_H=hp2, out_W=W2).check()
        P["wg2"].useful_M = B * H2 * W2
        # ---- conv3 forward (box): chunk = one tap x 64 channels; result goes to the PLAIN [B, H3*W3*64] matrix the Linear reads
        taps3 = [(kh, kw) for kh in range(k3) for kw in range(k3)]
        P["taps3"] = taps3
        P["fwd3"] = BoxGeometry(B=B, C=64, W=W2, hp_in=hp2, box_c=64, box_px=W2, box_h=hp2, row_step=1,
                                chunks=[(0, kw - p3, kh - p3 + 1 - 1) for kh, kw in taps3], hp_out=hp2, y0=1, y1=H2,
                                out_H=H3, out_W=W3, oy0=0)
        P["wg3"] = GatherGeometry(B=B, IH=hp2, IW=W2, C=64, OY=hp2, OX=W2, sy=1, sx=1, dy=[kh - p3 for kh, _ in taps3],
                                  dx=[kw - p3 for _, kw in taps3], out_H=hp2, out_W=W2).check()
        P["wg3"].useful_M = B * H2 * W2
        # ---- conv3 data gradient (box over the padded output gradient): flipped taps, written into act2's layout
        P["dg3"] = BoxGeometry(B=B, C=64, W=W2, hp_in=hp2, box_c=64, box_px=W2, box_h=hp2, row_step=1,
                               chunks=[(0, p3 - kw, p3 - kh) for kh, kw in taps3], hp_out=hp2, y0=1, y1=H2,
                               out_H=hp2, out_W=W2, oy0=1)
        # ---- conv2 data gradient: one box GEMM per stride phase over g2 (padded, real row i at i + 1), into act1's layout
        dg2 = []
        for py in range(2):
            for px in range(2):
                ny, nx = (H1 - py + 1) // 2, (W1 - px + 1) // 2
                taps = [(kh, kw) for kh in range(k2) if (py + p2 - kh) % 2 == 0 for kw in range(k2) if (px + p2 - kw) % 2 == 0]
                chunks = [(0, (px + p2 - kw) // 2, (py + p2 - kh) // 2 + 1) for kh, kw in taps]
                bh = min(hp2, 128 // nx)
                dg2.append((BoxGeometry(B=B, C=64, W=W2, hp_in=hp2, box_c=64, box_px=nx, box_h=bh, row_step=1, chunks=chunks,
                                        hp_out=hp2, y0=0, y1=ny - 1, out_H=hp1, out_W=W1, oys=2, oxs=2, oy0=py + off1, ox0=px,
                                        mask_W=W1p, mask_x0=xo1),
                            taps))
        P["dg2"] = dg2
        # ---- the same three stride-1 gathers in halo mode (activation tile resident, only the weights stream)
        full = dict(y1=H2, x1=W2 - 1, oy0=0, ox0=0)
        P["h_fwd3"] = HaloGeometry(B=B, W=W2, hp=hp2, halo_w=W2 + 2, halo_w0=-1, y0=1, N=c3.out_channels, out_H=H3, out_W=W3,
                                   subs=[dict(full, shifts=[(kh - p3, kw - p3) for kh, kw in taps3])])
        P["h_dg3"] = HaloGeometry(B=B, W=W2, hp=hp2, halo_w=W2 + 2, halo_w0=-1, y0=1, N=c2.out_channels, out_H=hp2, out_W=W2,
                                  subs=[dict(full, oy0=1, shifts=[(p3 - kh, p3 - kw) for kh, kw in taps3])])
        subs2 = [dict(shifts=[(ch[2], ch[1]) for ch in bg.chunks], y1=bg.y1, x1=bg.box_px - 1, oy0=bg.oy0, ox0=bg.ox0) for bg, _ in dg2]
        P["h_dg2"] = None
        if len(subs2) <= 4 and len({len(sb["shifts"]) for sb in subs2}) == 1 and len(subs2) * len(subs2[0]["shifts"]) <= 16:
            P["h_dg2"] = HaloGeometry(B=B, W=W2, hp=hp2, halo_w=W2 + 2, halo_w0=-1, y0=0, N=c1.out_channels, out_H=hp1, out_W=W1,
                                      oys=2, oxs=2, same_cols=True, mask_W=W1p, mask_x0=xo1, subs=subs2)
        if self.fc is not None:
            N, K = self.fc.weight.shape
            assert K == H3 * W3 * c3.out_channels
            P["fc"] = dict(N=N, K=K, fwd=linear_geometry(B, K), dgrad=linear_geometry(B, N), C=c3.out_channels, KH=H3, KW=W3)
        self._plans[B] = P
        return P

    def _buffers(self, B, like, keep=True):
        """Persistent zero-initialised padded tensors of batch size B.  ``keep=False``: a second set for inference calls
        (rollout / target / double-Q forwards under no_grad), so that they never overwrite the activations a pending
        backward of the SAME encoder still needs (act1 / act2 are both layer outputs and saved activations)."""
        key = ("buf", B) if keep else ("buf_inference", B)
        if key not in self._plans:
            P, be = self._plan(B), self.be
            z = lambda *shape: torch.zeros((be.planes,) + shape, dtype=torch.bfloat16, device=like.device)
            pairs = lambda t: t.view(be.planes, B * P["hp1"], P["W1p"] // 2, 2 * P["N1"])
            self._plans[key] = dict(act1=z(B * P["hp1"], P["W1p"], P["N1"]), act2=z(B * P["hp2"], P["W2"], P["N2"]),
                                    g3=z(B * P["hp2"], P["W2"], P["N3"]), g2=z(B * P["hp2"], P["W2"], P["N2"]),
                                    g1=z(B * P["hp1"], P["W1"], P["N1"]))
            self._plans[key]["act1_pairs"] = pairs(self._plans[key]["act1"])
        return self._plans[key]

    def _operands(self, P, scale):
        """Every weight operand form of one update in ONE launch (xb_pack_weights): forward packs, the Linear layer's
        transposed pack, the data-gradient matrices of conv3 and of conv2's four stride phases."""
        c1, c2, c3 = self.convs
        F, T, D = _lib.PACK_FORWARD, _lib.PACK_TRANSPOSED, _lib.PACK_DGRAD
        jobs = [(c1.weight.detach(), F, None, scale), (c2.weight.detach(), F, None, 1.0), (c3.weight.detach(), F, None, 1.0),
                (c3.weight.detach(), D, P["taps3"], 1.0)] + [(c2.weight.detach(), D, taps, 1.0) for _, taps in P["dg2"]]
        if self.fc is not None:
            F_ = P["fc"]
            w4 = self.fc.weight.detach().view(F_["N"], F_["C"], F_["KH"], F_["KW"])
            jobs += [(w4, F, None, 1.0), (w4, T, None, 1.0)]
        outs = pack_weights(jobs, self.be.planes, c1.weight.device)
        n2 = len(P["dg2"])
        ops = dict(w1=outs[0], w2=outs[1], w3=outs[2], wd3=outs[3], wd2=outs[4:4 + n2])
        if HALO and P["h_dg2"] is not None:
            ops["wd2_all"] = torch.cat(ops["wd2"], 1)             # the phases' matrices stacked as the sub-items' weight rows
        if self.fc is not None:
            ops.update(wfc=outs[4 + n2], wfc_t=outs[5 + n2])
        return ops

    def forward(self, x_pl, B, keep=True):
        """``keep=False`` (inference under no_grad): own activation buffers, ``_saved`` untouched."""
        be, P = self.be, self._plan(B)
        buf = self._buffers(B, x_pl, keep)
        c1, c2, c3 = self.convs
        raw = x_pl.shape[0] == 1 and be.planes > 1
        scale = 1.0 / 255.0 if raw else 1.0
        ops = self._operands(P, scale)
        gemm_gather(x_pl, ops["w1"], P["fwd1"], bias=c1.bias.detach(), relu=True, out_pl=buf["act1"], out_ld=P["N1"])
        gemm_box(buf["act1_pairs"], ops["w2"], P["fwd2"], bias=c2.bias.detach(), relu=True, out_pl=buf["act2"], out_ld=P["N2"])
        n3 = P["H2"] * P["W2"]
        act3 = be.empty_planes((B * n3, P["N3"]), x_pl)
        last_conv = self.fc is None
        out3 = be.empty_f32((B * n3, P["N3"]), x_pl) if last_conv else None
        (gemm_halo if HALO3 else gemm_box)(buf["act2"], ops["w3"], P["h_fwd3"] if HALO3 else P["fwd3"], bias=c3.bias.detach(), relu=True,
                                          out_pl=act3, out_f32=out3, out_ld=P["N3"])
        saved = dict(x=x_pl, act3=act3, scale=scale, ops=ops)
        if last_conv:
            if keep:
                self._saved = (B, saved)
            return out3
        F_ = P["fc"]
        y = be.empty_planes((B, F_["N"]), x_pl)
        out = be.empty_f32((B, F_["N"]), x_pl)
        gemm_gather(act3.view(be.planes, B, F_["K"]), ops["wfc"], F_["fwd"], bias=self.fc.bias.detach(), relu=True, out_f32=out, out_pl=y)
        saved.update(y=y)
        if keep:
            self._saved = (B, saved)
        return out

    @staticmethod
    def _into(p):
        """Where a parameter's gradient goes: straight into an existing contiguous float32 ``.grad`` (added, as autograd's
        accumulation would - the flat gradient bucket of the fused optimizer), else a fresh tensor returned to autograd."""
        g = p.grad
        if g is not None and g.is_contiguous() and g.dtype == torch.float32 and g.device == p.device:
            return dict(out=g, accumulate=True)
        return dict(out=None, accumulate=False)

    def backward(self, dz):
        be = self.be
        B, sv = self._saved
        P, buf = self._plan(B), self._buffers(B, dz)
        c1, c2, c3 = self.convs
        ops = sv["ops"]
        act3 = sv["act3"]
        ret = lambda p, t: None if p.grad is not None and t.data_ptr() == p.grad.data_ptr() else t.view_as(p)
        if self.fc is not None:
            F_ = P["fc"]
            g4 = be.split(dz * (sv["y"][0] > 0).to(dz.dtype))
            x3 = act3.view(be.planes, B, F_["K"])
            dwfc = be.wgrad(x3, g4, F_["fwd"], F_["N"], F_["C"], F_["KH"], F_["KW"], **self._into(self.fc.weight))
            dbfc = be.colsum(g4)
            if self._into(self.fc.bias)["accumulate"]:
                self.fc.bias.grad.add_(dbfc)
                dbfc = self.fc.bias.grad
            gfc = [ret(self.fc.weight, dwfc), ret(self.fc.bias, dbfc)]
            if self.grads_ready is not None and gfc[0] is None and gfc[1] is None:
                # the Linear layer's gradients (and those of everything after the encoder) are final and in place while the
                # whole convolution backward is still ahead: a sharded learner starts reducing them now
                self.grads_ready(self.fc.weight)
            # the Linear layer's data gradient lands straight in conv3's PADDED output-gradient tensor: image b's 6400 values
            # are rows 1 .. H2 of its hp2 rows (a matrix with hp2*W2*N3 elements per row, from column W2*N3); the mask is
            # the plain [B, 6400] activation; the column sums per (h, w, c) are conv3's bias-gradient partials
            ld3 = P["hp2"] * P["W2"] * P["N3"]
            cs3 = torch.empty((-(-B // 128), F_["K"]), dtype=torch.float32, device=dz.device)
            gemm_gather(g4, ops["wfc_t"], F_["dgrad"], out_pl=buf["g3"].view(be.planes, B, ld3), out_ld=ld3, out_c0=P["W2"] * P["N3"],
                        relu_mask=x3[0], mask_ld=F_["K"], mask_c0=0, colsum=cs3)
            db3 = bias_grad(cs3, P["N3"], **self._into(c3.bias))
        else:
            gfc = []
            g3p = be.split(dz * (act3[0] > 0).to(dz.dtype)).view(be.planes, B, P["H2"], P["W2"] * P["N3"])
            buf["g3"].view(be.planes, B, P["hp2"], P["W2"] * P["N3"])[:, :, 1:1 + P["H2"]].copy_(g3p)
            db3 = be.colsum(g3p.view(be.planes, -1, P["N3"]))
        g3 = buf["g3"]                                                     # conv3's output gradient, rows 1 .. H2 of hp2
        k3 = c3.kernel_size[0]
        if BOX_WGRAD3:
            sp3 = wgrad_box_splits(B * P["hp2"], 6, P["fwd3"].K, P["N3"])
            dw3 = wgrad_reduce(wgrad_box(buf["act2"], g3, P["fwd3"], 6, sp3), P["N3"], P["N2"], k3, k3, **self._into(c3.weight))
        else:
            dw3 = be.wgrad(buf["act2"], g3.view(be.planes, -1, P["N3"]), P["wg3"], P["N3"], P["N2"], k3, k3, **self._into(c3.weight))
        dg3 = P["h_dg3"] if HALO3 else P["dg3"]
        cs2 = torch.empty((dg3.m_tiles, P["N2"]), dtype=torch.float32, device=dz.device)
        (gemm_halo if HALO3 else gemm_box)(g3, ops["wd3"], dg3, out_pl=buf["g2"], out_ld=P["N2"], relu_mask=buf["act2"][0], colsum=cs2)
        db2 = bias_grad(cs2, P["N2"], **self._into(c2.bias))
        G2 = buf["g2"].view(be.planes, -1, P["N2"])
        k2 = c2.kernel_size[0]
        if BOX_WGRAD2:
            sp2 = wgrad_box_splits(B * P["hp2"], 6, P["fwd2"].K, P["N2"])
            dw2 = wgrad_reduce(wgrad_box(buf["act1_pairs"], buf["g2"], P["fwd2"], 6, sp2), P["N2"], P["N1"], k2, k2,
                               **self._into(c2.weight))
        else:
            dw2 = be.wgrad(buf["act1"], G2, P["wg2"], P["N2"], P["N1"], k2, k2, **self._into(c2.weight))
        if "wd2_all" in ops:
            cs1 = torch.empty((P["h_dg2"].m_tiles, P["N1"]), dtype=torch.float32, device=dz.device)
            gemm_halo(buf["g2"], ops["wd2_all"], P["h_dg2"], out_pl=buf["g1"], out_ld=P["N1"], relu_mask=buf["act1"][0], colsum=cs1)
        else:
            cs1 = torch.empty((sum(bg.m_tiles for bg, _ in P["dg2"]), P["N1"]), dtype=torch.float32, device=dz.device)
            row = 0
            for (bg, _), wd in zip(P["dg2"], ops["wd2"]):
                gemm_box(buf["g2"], wd, bg, out_pl=buf["g1"], out_ld=P["N1"], relu_mask=buf["act1"][0], colsum=cs1[row:row + bg.m_tiles])
                row += bg.m_tiles
        db1 = bias_grad(cs1, P["N1"], **self._into(c1.bias))
        G1 = buf["g1"].view(be.planes, -1, P["N1"])
        k1 = c1.kernel_size[0]
        dw1 = be.wgrad(sv["x"], G1, P["wg1"], P["N1"], self.in_hwc[2], k1, k1, sv["scale"], **self._into(c1.weight))
        convs = [ret(p, t) for p, t in ((c1.weight, dw1), (c1.bias, db1), (c2.weight, dw2), (c2.bias, db2), (c3.weight, dw3),
                                        (c3.bias, db3))]
        return convs + gfc


class _TCEncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, enc, x_pl, B, *params):
        ctx.enc = enc
        return enc.forward(x_pl, B)

    @staticmethod
    def backward(ctx, dz):
        return (None, None, None, *ctx.enc.backward(dz.contiguous()))


def tc_encode(enc, x_pl, B):
    """Differentiable call of a ``TensorCoreNatureCNN``: gradients reach the conv / linear parameters."""
    return _TCEncoderFn.apply(enc, x_pl, B, *enc.parameters())

"""Teacher-forced float64 checker of an assembled K12 encoder (``BoxNatureCNN`` or ``TensorCoreNatureCNN``,
xuance_b200/torch/utils/tc_conv.py) after one ``forward`` and one ``backward``.

Every layer is compared with float64 computed from the encoder's OWN stored input to that layer (the bf16 planes it keeps
between layers, summed in float64), and every data gradient from the encoder's own stored output gradient of the layer
above, masked exactly as the kernels mask (plane 0 of the saved activation > 0).  So no ReLU decision of the reference can
differ from the kernel's and every comparison is elementwise:

    forward   act1 = relu(conv1(x)),  act2 = relu(conv2(act1_k)),  act3 = relu(conv3(act2_k)),  z, y = relu(fc(act3_k))
    backward  g3 = ((dz * [y_k > 0]) @ W_fc) * [act3_k > 0],  g2 = conv3^T(g3_k) * [act2_k > 0],  g1 = conv2^T(g2_k) * [act1_k > 0]
              dW, db of every layer from that layer's kernel input and kernel output gradient

(_k = the kernel's stored value in float64; Basic_CNN has no fc: g3 = dz * [act3_k > 0]).

Bounds.  A compared element r = sum_k a_k w_k (+ bias) gets the bound

    |kernel - r|  <=  2^-23 * T  +  (c_rep + n * 2^-29 + m * 2^-24) * sum_k |a_k| |w_k|  +  2^-(8P) * |r|

with sum_k |a_k| |w_k| computed in float64 as the same operation on |a| and |w| (conv(|x|, |w|), |g| @ |W|, ...):
  * T: the tensor core adds each 16-deep block of products into a float32 accumulator with truncation (DESIGN.md
    section 4), which loses less than one ulp (2^-23 relative) of the largest of the accumulator before the add, the
    accumulator after it and the block's products.  For the forward and data-gradient GEMMs T is computed in float64
    along the kernels' own K order ((kh, kw, c) of the packed weights, the taps of a data-gradient phase in the order the
    plan lists them, (h, w, c) for the Linear layer): T = sum over 16-deep steps j of max(|S_{j-1}|, |S_j|,
    sum_{k in j} |a_k w_k|), S_j the exact partial sum after step j.  For a weight gradient the chain runs over sites in
    an order set by the split rule, and T is bounded by n * sum_k |a_k| |w_k| with n = the sites of one split / 16
    (``wgrad_splits`` / ``wgrad_box_splits``; 60-site box chunks take 4 steps).
  * n * 2^-29: the lower plane-product groups (2^-8 and smaller) have their own truncating chains, and the hi.hi
    accumulator the truncation acts on differs from S_j by those groups: below 2^-6 of one ulp per step.
  * c_rep = (P + 2) * 2^-(8P): an operand of P planes is exact to 2^-(8P) of its value (each plane is the bf16 rounding of
    the residual the planes before it leave, 8 bits each); a launch drops the plane products whose indices sum to >= P,
    P - 1 products of order 2^-(8P); the weight's residual adds one more 2^-(8P); float32 rounding of the 1/255 folded into
    conv1's weights and of the bias add are below 2^-(8P) for P <= 3.  The activations the kernels read are the stored
    planes themselves, so they carry no representation error here.
  * m * 2^-24: round-to-nearest float32 additions after the accumulators: the plane groups added in the epilogue (P), the
    split partials in xb_wgrad_reduce (its fold of groups of splits, then the groups), the 1/255 scale, the column sums
    of a bias gradient (128 rows of a tile in any order, then the tiles), torch's float32 column sums (rows, any order).
  * 2^-(8P) * |r|: the compared tensor itself stored as P bf16 planes (none for the float32 outputs).

Storage.  A rounding bound cannot tell a tensor stored with a plane too few (a change of up to 2^-(8P-6) |r|) from the
accumulation error, so the stored planes are checked on their own: with three planes every float32 is exact, and the
planes of each stored tensor must be bitwise the three-plane split of their own float32 sum; y (the Linear layer's
planes) must be bitwise the split of the float32 output z of the same epilogue (conv3's planes of Basic_CNN likewise);
and the last plane must really be written: it is zero only where the float32 value fits in the planes before it (about
one value in 2^8 for the last of three planes, 2^16 for the last of two), so at most 1/16 of the non-zero values of a
stored tensor may have a zero last plane.

``check`` returns {tensor: max(|kernel - r| / bound)} and raises on any ratio > 1 and on any padding element of the
persistent padded buffers that is not bitwise zero.

The weight- and bias-gradient bounds above are worst cases over chains of up to 4096 sites and leave room for a lost or
repeated chunk, split or column-sum row at large B; tests/test_gpu_k12_exact_reductions.py (with tests/k12_exact_refs.py)
pins those reductions bit for bit on exactly representable operands instead.
"""
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from xuance_b200.torch.utils import tc_conv as tc

U_TRUNC = 2.0 ** -23
U_RN = 2.0 ** -24


class RecordingBackend(tc.CudaBackend):
    """``CudaBackend`` that keeps the (input planes, output-gradient planes) of the weight gradients of the latest
    backward (at most four layers, in backward order): ``TensorCoreNatureCNN`` does not keep its data gradients."""

    def __init__(self, planes=3):
        super().__init__(planes)
        self.wgrads = []

    def wgrad(self, x_pl, g_pl, geom, N, C, KH, KW, scale=1.0, out=None, accumulate=False):
        self.wgrads = (self.wgrads + [(x_pl, g_pl, geom)])[-4:]
        return super().wgrad(x_pl, g_pl, geom, N, C, KH, KW, scale=scale, out=out, accumulate=accumulate)


def _f64(pl):
    return pl.double().sum(0)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def reduce_chain(splits):
    """Float32 additions on the longest path of xb_wgrad_reduce for ``splits`` partial rows (fold groups first above 256)."""
    if splits > 256:
        group = -(-splits // 128)
        return group + -(-splits // group)
    return splits


def _gather_steps(M, K, N, planes):
    """16-site steps of one split of the gathered weight gradient (CudaBackend.wgrad's split rule) and the split count."""
    s = tc.wgrad_splits(M, K, N // tc.n_tile_for(N, planes))
    per = -(-(-(-M // s)) // tc.KC) * tc.KC
    return per // 16, s


def _box_steps(g_rows, K, N, spr=10, box_h=6):
    s = tc.wgrad_box_splits(g_rows, box_h, K, N)
    per = -(-(-(-g_rows // s)) // box_h) * box_h
    return (per // box_h) * (-(-box_h * spr // 16)), s


def taps_matrix(x, OY, OX, s, offs):
    """A operand [B*OY*OX, T*C] of a convolution in the kernels' K order: tap t reads x[b, y*s + dy_t, x*s + dx_t, :]
    (NHWC, zero outside the image), taps in the order of ``offs``."""
    B, H, W, C = x.shape
    ys, xs = torch.arange(OY, device=x.device) * s, torch.arange(OX, device=x.device) * s
    cols = []
    for dy, dx in offs:
        iy, ix = ys + dy, xs + dx
        ok = ((iy >= 0) & (iy < H))[:, None] & ((ix >= 0) & (ix < W))[None, :]
        cols.append(x[:, iy.clamp(0, H - 1)][:, :, ix.clamp(0, W - 1)] * ok[None, :, :, None])
    return torch.cat(cols, -1).reshape(B * OY * OX, -1)


def trunc_chain(A, Wm):
    """T of the module docstring for D = A @ Wm^T (float64 [M, K] and [N, K], K in accumulation order): the sum over the
    16-deep steps of max(|S_{j-1}|, |S_j|, sum_{k in j} |a_k w_k|)."""
    S = torch.zeros(A.shape[0], Wm.shape[0], dtype=torch.float64, device=A.device)
    prev, acc = torch.zeros_like(S), torch.zeros_like(S)
    for k0 in range(0, A.shape[1], 16):
        a, w = A[:, k0:k0 + 16], Wm[:, k0:k0 + 16]
        S += a @ w.t()
        cur = S.abs()
        acc += torch.maximum(torch.maximum(prev, cur), a.abs() @ w.abs().t())
        prev = cur
    return acc


def conv_chain(x, Wm, OY, OX, s, offs, images=256):
    """trunc_chain of a convolution over NHWC x, in chunks of images; returns [B, OY, OX, N]."""
    return torch.cat([trunc_chain(taps_matrix(x[i:i + images], OY, OX, s, offs), Wm).view(-1, OY, OX, Wm.shape[0])
                      for i in range(0, x.shape[0], images)])


def _packed(w):
    """[N, C, KH, KW] -> [N, (kh, kw, c)] (the forward packs' column order)."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)


def check_storage(name, pl, f32=None):
    """The stored planes ``pl`` [P, ...] of one tensor: bitwise the split of their own float32 sum (three planes; with two
    the sum of the planes is not the float32 value the kernel split), bitwise the split of ``f32`` when the same
    epilogue also wrote the float32 value, and a last plane that is really written."""
    P = pl.shape[0]
    bits = lambda t: torch.where(t == 0, torch.zeros_like(t.view(torch.int16)), t.view(torch.int16))     # -0.0 as +0.0
    if f32 is not None:
        want = split_ref(f32.reshape(pl.shape[1:]), 3)[:P]
        assert torch.equal(bits(pl), bits(want)), "%s: planes are not the split of the float32 output" % name
    if P == 3:
        want = split_ref(pl.double().sum(0).float(), 3)
        assert torch.equal(bits(pl), bits(want)), "%s: planes are not the split of their own sum" % name
    if P > 1:
        nz = pl[0] != 0
        n_nz = int(nz.sum())
        empty = int((nz & (pl[P - 1] == 0)).sum())
        assert empty * 16 <= n_nz, "%s: the last of %d planes is zero on %d of %d non-zero values" % (name, P, empty, n_nz)


def split_ref(x, planes):
    """float32 -> bf16 planes, plane q = bf16 of the residual the planes before it leave (xb_split_bf16)."""
    r, out = x.float().clone(), []
    for _ in range(planes):
        h = r.bfloat16()
        out.append(h)
        r = r - h.float()
    return torch.stack(out)


def capture(enc, B, x_pl, z, grads):
    """Everything the checker compares, as float64 NHWC tensors, from either encoder class after forward + backward.
    ``grads``: the fresh gradients in ``enc.parameters()`` order."""
    Pn = enc.be.planes
    c = dict(B=B, P=Pn, raw=x_pl.shape[0] == 1 and Pn > 1, z=z.double(), z_raw=z, grads=[g.double() for g in grads])
    c["x"] = _f64(x_pl).reshape(B, *enc.in_hwc)
    c["scale"] = 1.0 / 255.0 if c["raw"] else 1.0
    if isinstance(enc, tc.BoxNatureCNN):
        P = enc._plan(B)
        buf = enc._plans[("buf", B)]
        _, sv = enc._saved
        H1, W1, H2, W2, off1, xo1 = P["H1"], P["W1"], P["H2"], P["W2"], P["off1"], P["xo1"]
        a1 = buf["act1"].view(Pn, B, P["hp1"], P["W1p"], P["N1"])[:, :, off1:off1 + H1, xo1:xo1 + W1]
        a2 = buf["act2"].view(Pn, B, P["hp2"], W2, P["N2"])[:, :, 1:1 + H2]
        a3 = sv["act3"].view(Pn, B, H2, W2, P["N3"])
        g3 = buf["g3"].view(Pn, B, P["hp2"], W2, P["N3"])[:, :, 1:1 + H2]
        g2 = buf["g2"].view(Pn, B, P["hp2"], W2, P["N2"])[:, :, 1:1 + H2]
        g1 = buf["g1"].view(Pn, B, P["hp1"], W1, P["N1"])[:, :, off1:off1 + H1]
        c["y"] = sv.get("y")
    else:
        _, saved = enc._saved
        plan = enc._plan(B)
        shp = [(L["fwd"].OY, L["fwd"].OX, L["N"]) for L in plan[:3]]
        a1, a2, a3 = (saved[i]["y"].view(Pn, B, *shp[i]) for i in range(3))
        c["y"] = saved[3]["y"] if enc.fc is not None else None
        gs = [g for _, g, _ in enc.be.wgrads[-len(plan):]][::-1]     # recorded in backward order: (fc,) conv3, conv2, conv1
        g1, g2, g3 = (gs[i].view(Pn, B, *shp[i]) for i in range(3))
    c["g1"], c["g2"], c["g3"] = _f64(g1), _f64(g2), _f64(g3)
    c["pl"] = dict(act1=a1, act2=a2, act3=a3, g3=g3, g2=g2, g1=g1)
    c["act1"], c["act2"], c["act3"] = _f64(a1), _f64(a2), _f64(a3)
    c["m1"], c["m2"], c["m3"] = a1[0] > 0, a2[0] > 0, a3[0] > 0
    if c["y"] is not None:
        c["pl"]["y"] = c["y"]
        c["my"] = c["y"][0] > 0
        c["y"] = _f64(c["y"])
    return c


class _Ratios(dict):
    def add(self, name, got, ref, mag, c, store, chain=None):
        err = (got.double() - ref).abs()
        bound = c * mag + store * ref.abs() + (U_TRUNC * chain if chain is not None else 0.0)
        bad = err > bound
        self[name] = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
        if bool(bad.any()):
            i = int(bad.reshape(-1).nonzero()[0])
            raise AssertionError("%s: |error| %.3g exceeds its bound %.3g at flat index %d (largest ratio %.3g)"
                                 % (name, float(err.reshape(-1)[i]), float(bound.reshape(-1)[i]), i, self[name]))


def check(enc, c, dz):
    """Compare the capture ``c`` of ``enc`` (forward of the planes ``c['x']`` and backward of ``dz``) with float64."""
    B, Pn = c["B"], c["P"]
    c1, c2, c3 = enc.convs
    fc = enc.fc
    d = lambda t: t.detach().double()
    rep = (Pn + 2) * 2.0 ** (-8 * Pn)
    store = 2.0 ** (-8 * Pn)
    ep = Pn + 2                                               # epilogue group adds, bias, 1/255
    r = _Ratios()
    box = isinstance(enc, tc.BoxNatureCNN)
    cf = lambda n, m=0: rep + n * U_TRUNC + (m + ep) * U_RN          # a chain bounded by n steps of sum |a||w|
    ct = lambda n, m=0: rep + n * U_TRUNC / 64 + (m + ep) * U_RN     # a chain T computed along the K order

    # ---- storage of every stored tensor
    for name, pl in c["pl"].items():
        f32 = c["z_raw"] if (name == "y" or (name == "act3" and fc is None)) else None
        check_storage(name, pl, f32)

    def fwd_chain(x, conv):
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        OY, OX = (x.shape[1] + 2 * p - k) // s + 1, (x.shape[2] + 2 * p - k) // s + 1
        return conv_chain(x, _packed(d(conv.weight)), OY, OX, s, [(kh - p, kw - p) for kh in range(k) for kw in range(k)])

    def conv_fwd(x, conv, relu=True):
        w, b = d(conv.weight), d(conv.bias)
        s, p = conv.stride, conv.padding
        ref = F.conv2d(_nchw(x), w, b, stride=s, padding=p)
        mag = F.conv2d(_nchw(x.abs()), w.abs(), b.abs(), stride=s, padding=p)
        return _nhwc(F.relu(ref) if relu else ref), _nhwc(mag)

    # ---- forward, layer by layer from the kernel's own inputs
    x_in = c["x"] * c["scale"]
    ref, mag = conv_fwd(x_in, c1)
    r.add("act1", c["act1"], ref, mag, ct(c1.weight[0].numel() // 16), store, fwd_chain(x_in, c1))
    ref, mag = conv_fwd(c["act1"], c2)
    r.add("act2", c["act2"], ref, mag, ct(c2.weight[0].numel() // 16), store, fwd_chain(c["act1"], c2))
    ref, mag = conv_fwd(c["act2"], c3)
    ch3 = fwd_chain(c["act2"], c3)
    r.add("act3", c["act3"], ref, mag, ct(c3.weight[0].numel() // 16), store, ch3)
    if fc is not None:
        a3 = _nchw(c["act3"]).reshape(B, -1)
        wf, bf = d(fc.weight), d(fc.bias)
        wf_k = _packed(wf.view(wf.shape[0], *_nchw(c["act3"]).shape[1:]))          # [N, (h, w, c)]: the kernel's K order
        ref = F.relu(a3 @ wf.t() + bf)
        mag = a3.abs() @ wf.abs().t() + bf.abs()
        chf = trunc_chain(c["act3"].reshape(B, -1), wf_k)
        cfc = ct(fc.weight.shape[1] // 16)
        r.add("z", c["z"], ref, mag, cfc, 0.0, chf)
        r.add("y", c["y"], ref, mag, cfc, store, chf)
    else:
        r.add("z", c["z"].view(c["act3"].shape), ref, mag, ct(c3.weight[0].numel() // 16), 0.0, ch3)

    # ---- backward: data gradients from the kernel's own output gradients, masked as the kernels mask
    dz = dz.double()
    grads = dict(zip(("w1", "b1", "w2", "b2", "w3", "b3", "wf", "bf"), c["grads"]))
    if fc is not None:
        gy = dz * c["my"]
        ref = _nhwc((gy @ wf).view(B, *_nchw(c["act3"]).shape[1:])) * c["m3"]
        mag = _nhwc((gy.abs() @ wf.abs()).view(B, *_nchw(c["act3"]).shape[1:]))
        chg = trunc_chain(gy, wf_k.t()).view(c["act3"].shape)                       # K order = the Linear's outputs
        r.add("g3", c["g3"], ref, mag, ct(fc.weight.shape[0] // 16), store, chg)
        n, s = _gather_steps(B, fc.weight.shape[1], fc.weight.shape[0], Pn)
        r.add("fc.weight", grads["wf"], gy.t() @ a3, gy.abs().t() @ a3.abs(), cf(n, reduce_chain(s)), 0.0)
        r.add("fc.bias", grads["bf"], gy.sum(0), gy.abs().sum(0), rep + (B + Pn) * U_RN, 0.0)
    else:
        gy = (dz.view(c["act3"].shape) * c["m3"])
        r.add("g3", c["g3"], gy, torch.zeros_like(gy), 0.0, store)
    g3 = c["g3"]

    def dgrad(g, x, conv, mask):
        w = d(conv.weight)
        kw = dict(stride=conv.stride, padding=conv.padding)
        ref = conv2d_input(_nchw(x).shape, w, _nchw(g), **kw)
        mag = conv2d_input(_nchw(x).shape, w.abs(), _nchw(g.abs()), **kw)
        return _nhwc(ref) * mask, _nhwc(mag)

    def wgrad(x, g, conv):
        w = conv.weight
        kw = dict(stride=conv.stride, padding=conv.padding)
        return (conv2d_weight(_nchw(x), w.shape, _nchw(g), **kw),
                conv2d_weight(_nchw(x.abs()), w.shape, _nchw(g.abs()), **kw))

    # data-gradient chains: conv3 as one stride-1 gather with flipped taps, conv2 as four stride phases (taps in plan order)
    k3, p3 = c3.kernel_size[0], c3.padding[0]
    taps3 = [(kh, kw) for kh in range(k3) for kw in range(k3)]
    ch = conv_chain(g3, tc.dgrad_weight_matrix(d(c3.weight), taps3), g3.shape[1], g3.shape[2], 1,
                    [(p3 - kh, p3 - kw) for kh, kw in taps3])
    ref, mag = dgrad(g3, c["act2"], c3, c["m2"])
    r.add("g2", c["g2"], ref, mag, ct(c3.weight.shape[0] * 9 // 16), store, ch)
    H1, W1 = c["act1"].shape[1:3]
    ch = torch.zeros_like(c["g1"])
    k2, s2, p2 = c2.kernel_size[0], c2.stride[0], c2.padding[0]
    for geom, taps in tc.conv_dgrad_geometries(B, H1, W1, c2.in_channels, k2, k2, s2, p2, c2.out_channels):
        ch[:, geom.oy0::s2, geom.ox0::s2] = conv_chain(c["g2"], tc.dgrad_weight_matrix(d(c2.weight), taps), geom.OY, geom.OX, 1,
                                                      list(zip(geom.dy, geom.dx)))
    ref, mag = dgrad(c["g2"], c["act1"], c2, c["m1"])
    r.add("g1", c["g1"], ref, mag, ct(c2.weight.shape[0] * 4 // 16), store, ch)

    # ---- weight gradients: chain lengths of the path the encoder took
    if box:
        P = enc._plan(B)
        hp1, hp2, W1, W2 = P["hp1"], P["hp2"], P["W1"], P["W2"]
        n3, s3 = _box_steps(B * hp2, 576, 64) if tc.BOX_WGRAD3 else _gather_steps(B * hp2 * W2, 576, 64, Pn)
        n2, s2 = _box_steps(B * hp2, 512, 64) if tc.BOX_WGRAD2 else _gather_steps(B * hp2 * W2, 512, 64, Pn)
        n1, s1 = _gather_steps(B * hp1 * W1, c1.weight[0].numel(), 32, Pn)
        t3 = -(-B // 128) * (fc.weight.shape[1] // 64) if fc is not None else None
        t2 = P["h_dg3"].m_tiles if tc.HALO3 else P["dg3"].m_tiles
        t1 = P["h_dg2"].m_tiles if (tc.HALO and P["h_dg2"] is not None) else sum(bg.m_tiles for bg, _ in P["dg2"])
        bias_c = lambda t: rep + (128 + reduce_chain(t) + ep) * U_RN
        cb3 = bias_c(t3) if t3 is not None else rep + (g3[..., 0].numel() + Pn) * U_RN
        cb2, cb1 = bias_c(t2), bias_c(t1)
    else:
        n3, s3 = _gather_steps(B * 100, 576, 64, Pn)
        n2, s2 = _gather_steps(B * 100, 512, 64, Pn)
        n1, s1 = _gather_steps(B * 441, c1.weight[0].numel(), 32, Pn)
        rows = lambda g: rep + (g.shape[0] * g.shape[1] * g.shape[2] + Pn) * U_RN
        cb3, cb2, cb1 = rows(g3), rows(c["g2"]), rows(c["g1"])
    ref, mag = wgrad(c["act2"], g3, c3)
    r.add("conv3.weight", grads["w3"], ref, mag, cf(n3, reduce_chain(s3)), 0.0)
    r.add("conv3.bias", grads["b3"], g3.sum((0, 1, 2)), g3.abs().sum((0, 1, 2)), cb3 + store, 0.0)
    ref, mag = wgrad(c["act1"], c["g2"], c2)
    r.add("conv2.weight", grads["w2"], ref, mag, cf(n2, reduce_chain(s2)), 0.0)
    r.add("conv2.bias", grads["b2"], c["g2"].sum((0, 1, 2)), c["g2"].abs().sum((0, 1, 2)), cb2 + store, 0.0)
    ref, mag = wgrad(x_in, c["g1"], c1)
    r.add("conv1.weight", grads["w1"], ref, mag, cf(n1, reduce_chain(s1)), 0.0)
    r.add("conv1.bias", grads["b1"], c["g1"].sum((0, 1, 2)), c["g1"].abs().sum((0, 1, 2)), cb1 + store, 0.0)
    return dict(r)


def padding_regions(enc, B, kind="buf"):
    """The padding elements of the five persistent padded tensors of a ``BoxNatureCNN`` at batch size B (bool masks);
    ``kind`` "buf_inference": the set the keep=False (no_grad) forwards use."""
    P = enc._plan(B)
    buf = enc._plans[(kind, B)]
    out = {}
    for name, hp, W, lo, hi, x0, x1 in (("act1", P["hp1"], P["W1p"], P["off1"], P["off1"] + P["H1"], P["xo1"], P["xo1"] + P["W1"]),
                                         ("act2", P["hp2"], P["W2"], 1, 1 + P["H2"], 0, P["W2"]),
                                         ("g3", P["hp2"], P["W2"], 1, 1 + P["H2"], 0, P["W2"]),
                                         ("g2", P["hp2"], P["W2"], 1, 1 + P["H2"], 0, P["W2"]),
                                         ("g1", P["hp1"], P["W1"], P["off1"], P["off1"] + P["H1"], 0, P["W1"])):
        t = buf[name]
        v = t.view(t.shape[0], B, hp, W, t.shape[-1])
        pad = torch.ones((hp, W), dtype=torch.bool, device=t.device)
        pad[lo:hi, x0:x1] = False
        out[name] = (v, pad)
    return out


def check_padding(enc, B, kind="buf"):
    """Every padding element of act1, act2, g3, g2, g1 is bitwise zero (+0.0 in every plane)."""
    for name, (v, pad) in padding_regions(enc, B, kind).items():
        bits = v.view(torch.int16)[:, :, pad]
        nz = int((bits != 0).sum())
        assert nz == 0, "%s: %d padding elements are not +0.0" % (name, nz)

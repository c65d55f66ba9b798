"""Host logic of K12's padded-row / TMA-box / halo modes (CPU): the geometry tables BoxNatureCNN builds are executed by a NumPy
restatement of what include/xb200.h says xb_gemm_box_tc / xb_gemm_halo_tc compute, and compared with torch convolutions and
their autograd.  The CUDA kernels are pinned against the same float64 references in tests/test_gpu_tc_conv.py; this file pins
the tables themselves (chunk order, pixel-pair view, row phases, shifts, valid extents, output placement)."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from xuance_b200.torch.utils import tc_conv as tc


def _plan(B):
    torch.manual_seed(3)
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    enc = tc.BoxNatureCNN(convs, None, (84, 84, 4), backend=tc.CudaBackend(3))
    assert enc._box_ok()
    return convs, enc._plan(B)


def box_gemm(x, w, bg, out, N, relu=False, mask=None):
    """xb_gemm_box_tc in NumPy.  x [B*hp_in, W, C] float64, w [N, n_chunks*64]; writes into out [B*out_H, out_W, N]."""
    rows, W, C = x.shape
    for R in range(bg.B * bg.hp_out):
        b, y = divmod(R, bg.hp_out)
        if not (bg.y0 <= y <= bg.y1):
            continue
        for xs in range(bg.box_px):
            a = np.zeros(64 * len(bg.chunks))
            for i, (c0, w0, r0) in enumerate(bg.chunks):
                row, px = R * bg.row_step + r0, w0 + xs
                if 0 <= row < rows and 0 <= px < W:
                    a[64 * i:64 * i + 64] = x[row, px, c0:c0 + 64]
            v = w @ a
            if relu:
                v = np.maximum(v, 0.0)
            orow, ocol = b * bg.out_H + (y - bg.y0) * bg.oys + bg.oy0, xs * bg.oxs + bg.ox0
            if mask is not None:
                v = v * (mask[orow, ocol + bg.mask_x0] > 0)
            out[orow, ocol] = v


def halo_gemm(x, w, hg, out, mask=None):
    """xb_gemm_halo_tc in NumPy.  x [B*hp, W, 64]; w [n_sub*N, n_chunks*64]; out [B*out_H, out_W, N (same_cols) or n_sub*N]."""
    rows, W, _ = x.shape
    for R in range(hg.B * hg.hp):
        b, y = divmod(R, hg.hp)
        for hc in range(hg.halo_w):
            px = hc + hg.halo_w0
            for j, sb in enumerate(hg.subs):
                if not (hg.y0 <= y <= sb["y1"] and 0 <= px <= sb["x1"]):
                    continue
                a = np.zeros(64 * hg.n_chunks)
                for i, (dr, dc) in enumerate(sb["shifts"]):
                    assert hg.halo_w0 <= px + dc <= hg.halo_w0 + hg.halo_w - 1, "a tap of a valid site leaves its raster row"
                    if 0 <= R + dr < rows and 0 <= px + dc < W:
                        a[64 * i:64 * i + 64] = x[R + dr, px + dc]
                v = w[j * hg.N:(j + 1) * hg.N] @ a
                orow, ocol = b * hg.out_H + (y - hg.y0) * hg.oys + sb["oy0"], px * hg.oxs + sb["ox0"]
                if mask is not None:
                    v = v * (mask[orow, ocol + hg.mask_x0] > 0)
                c0 = 0 if hg.same_cols else j * hg.N
                out[orow, ocol, c0:c0 + hg.N] = v


def packed(wt):
    """torch conv weight [N, C, KH, KW] -> [N, (kh, kw, c)] (xb_pack_conv_weight order)."""
    return wt.permute(0, 2, 3, 1).reshape(wt.shape[0], -1).double().numpy()


def test_box_and_halo_tables_compute_the_convolutions():
    B = 2
    convs, P = _plan(B)
    hp1, hp2, off1, W1p, xo1 = P["hp1"], P["hp2"], P["off1"], P["W1p"], P["xo1"]
    w2, b2, w3 = convs[1].weight.detach(), convs[1].bias.detach(), convs[2].weight.detach()
    rng = np.random.default_rng(0)
    a1 = rng.standard_normal((B, 21, 21, 32))
    act1 = np.zeros((B, hp1, W1p, 32))
    act1[:, off1:off1 + 21, xo1:xo1 + 21] = a1
    # conv2 forward: TMA boxes over the pixel-pair view, row phases
    pairs = act1.reshape(B * hp1, W1p // 2, 64)
    out2 = np.zeros((B * hp2, 10, 64))
    box_gemm(pairs, packed(w2), P["fwd2"], out2, 64)
    t = lambda a: torch.from_numpy(a).permute(0, 3, 1, 2)
    want2 = F.conv2d(t(a1), w2.double(), None, stride=2, padding=1).permute(0, 2, 3, 1).numpy()
    got2 = out2.reshape(B, hp2, 10, 64)
    np.testing.assert_allclose(got2[:, 1:11], want2, atol=1e-10)
    assert np.abs(got2[:, 0]).max() == 0 and np.abs(got2[:, 11]).max() == 0
    # conv3 forward: box and halo tables
    a2 = rng.standard_normal((B, 10, 10, 64))
    act2 = np.zeros((B, hp2, 10, 64))
    act2[:, 1:11] = a2
    act2 = act2.reshape(B * hp2, 10, 64)
    want3 = F.conv2d(t(a2), w3.double(), None, stride=1, padding=1).permute(0, 2, 3, 1).numpy()
    for fn, geo in ((box_gemm, P["fwd3"]), (halo_gemm, P["h_fwd3"])):
        out3 = np.zeros((B * 10, 10, 64))
        fn(act2, packed(w3), geo, out3) if fn is halo_gemm else fn(act2, packed(w3), geo, out3, 64)
        np.testing.assert_allclose(out3.reshape(B, 10, 10, 64), want3, atol=1e-10)
    # conv3 data gradient (flipped taps), box and halo, with the ReLU mask of act2
    g3 = rng.standard_normal((B, 10, 10, 64))
    g3p = np.zeros((B, hp2, 10, 64))
    g3p[:, 1:11] = g3
    g3p = g3p.reshape(B * hp2, 10, 64)
    x2 = t(a2).requires_grad_(True)
    (dx2,) = torch.autograd.grad(F.conv2d(x2, w3.double(), stride=1, padding=1), x2, t(g3))
    mask2 = act2.reshape(B * hp2, 10, 64)
    want_d2 = dx2.permute(0, 2, 3, 1).numpy() * (a2 > 0)
    wd3 = tc.dgrad_weight_matrix(w3, P["taps3"]).double().numpy()
    for fn, geo in ((box_gemm, P["dg3"]), (halo_gemm, P["h_dg3"])):
        d2 = np.zeros((B * hp2, 10, 64))
        fn(g3p, wd3, geo, d2, mask=mask2) if fn is halo_gemm else fn(g3p, wd3, geo, d2, 64, mask=mask2)
        np.testing.assert_allclose(d2.reshape(B, hp2, 10, 64)[:, 1:11], want_d2, atol=1e-10)
    # conv2 data gradient: four stride phases (four box launches / one halo launch), mask = act1 in its wider layout
    g2 = rng.standard_normal((B, 10, 10, 64))
    g2p = np.zeros((B, hp2, 10, 64))
    g2p[:, 1:11] = g2
    g2p = g2p.reshape(B * hp2, 10, 64)
    x1 = t(a1).requires_grad_(True)
    (dx1,) = torch.autograd.grad(F.conv2d(x1, w2.double(), stride=2, padding=1), x1, t(g2))
    want_d1 = dx1.permute(0, 2, 3, 1).numpy() * (a1 > 0)
    mask1 = act1.reshape(B * hp1, W1p, 32)
    d1 = np.zeros((B * hp1, 21, 32))
    for bg, taps in P["dg2"]:
        box_gemm(g2p, tc.dgrad_weight_matrix(w2, taps).double().numpy(), bg, d1, 32, mask=mask1)
    np.testing.assert_allclose(d1.reshape(B, hp1, 21, 32)[:, off1:off1 + 21], want_d1, atol=1e-10)
    d1h = np.zeros((B * hp1, 21, 32))
    wd2_all = np.concatenate([tc.dgrad_weight_matrix(w2, taps).double().numpy() for _, taps in P["dg2"]], 0)
    halo_gemm(g2p, wd2_all, P["h_dg2"], d1h, mask=mask1)
    np.testing.assert_allclose(d1h.reshape(B, hp1, 21, 32)[:, off1:off1 + 21], want_d1, atol=1e-10)
    assert np.abs(d1h.reshape(B, hp1, 21, 32)[:, :off1]).max() == 0


def test_halo_tile_holds_every_tap_of_its_128_positions():
    """The resident tile of M tile t starts at row floor((128 t + lo) / halo_w) and has the rows xb_gemm_halo_tc allocates:
    every (position + shift) of the tile must fall inside it (the kernel reads it through a descriptor offset)."""
    _, P = _plan(5)
    for key in ("h_fwd3", "h_dg3", "h_dg2"):
        hg = P[key]
        shifts = [dr * hg.halo_w + dc for sb in hg.subs for dr, dc in sb["shifts"]]
        lo, hi = min(0, min(shifts)), max(0, max(shifts))
        halo_rows = (hg.halo_w - 1 + 128 + hi - lo + hg.halo_w - 1) // hg.halo_w
        assert halo_rows * hg.halo_w * 128 * 3 * 2 + 2 * 3 * hg.N * 128 <= 212 * 1024        # two tiles + two ring stages fit
        for tile in range(-(-hg.M // 128)):
            r_lo = (tile * 128 + lo) // hg.halo_w
            s0 = tile * 128 - r_lo * hg.halo_w
            assert 0 <= s0 + lo and s0 + hi + 127 < halo_rows * hg.halo_w, (key, tile)


# ------------------------------------------------------------------------------------------------ the assembled encoder
# NumPy / torch restatements of the module functions BoxNatureCNN.forward / .backward call, in float64 with the kernels'
# output formats (float32 rows, bf16 planes of the float32 result, per-tile column sums, [splits, K, N] partials), so that
# the orchestration - persistent padded buffers, output placements, masks, column-sum row counts, accumulation into
# ``.grad`` - runs on the CPU and is checked by the same teacher-forced float64 checker as the GPU encoder
# (tests/k12_encoder_refs.py).
def _planes_ref(x, planes):
    r, out = x.float().clone(), []
    for _ in range(planes):
        h = r.bfloat16()
        out.append(h)
        r = r - h.float()
    return torch.stack(out)


def r_split_bf16(x, planes=2):
    return _planes_ref(x.contiguous(), planes)


def r_pack_weights(jobs, planes, device):
    from xuance_b200 import _lib
    outs = []
    for w, mode, taps, scale in jobs:
        N = w.shape[0]
        if mode == _lib.PACK_DGRAD:
            m = tc.dgrad_weight_matrix(w.float(), taps)
        else:
            m = w.float().permute(0, 2, 3, 1).reshape(N, -1) * np.float32(scale)
            m = m.t() if mode == _lib.PACK_TRANSPOSED else m
        outs.append(_planes_ref(m.contiguous(), planes))
    return outs


def r_pack_conv_weight(w, planes=2, scale=1.0):
    return _planes_ref(w.float().permute(0, 2, 3, 1).reshape(w.shape[0], -1) * np.float32(scale), planes)


def _epilogue(v, opix, mpix, tile, bias, relu, out_f32, out_pl, out_ld, out_c0, mask, mask_ld, mask_c0, colsum):
    """v [rows, N] float64 of the rows a launch writes; opix / mpix their output / mask pixels, tile their colsum row."""
    N = v.shape[1]
    cols = torch.arange(N, device=v.device)
    if bias is not None:
        v = v + bias.double()
    if relu:
        v = v.clamp_min(0.0)
    if mask is not None:
        keep = mask.reshape(-1)[(mpix * mask_ld + mask_c0)[:, None] + cols].float() > 0
        v = torch.where(keep, v, torch.zeros_like(v))
    v = v.float()
    idx = (opix * out_ld + out_c0)[:, None] + cols
    if out_f32 is not None:
        out_f32.view(-1)[idx] = v
    if out_pl is not None:
        pl = _planes_ref(v, 3)
        for q in range(out_pl.shape[0]):
            out_pl[q].view(-1)[idx] = pl[q]
    if colsum is not None:
        cs = torch.zeros(colsum.shape[0], N, dtype=torch.float64, device=v.device)
        cs.index_add_(0, tile, v.double())
        colsum.view(-1, N).copy_(cs.float())


def _gathered(x_pl, g):
    """The [M, T*C] A operand of the gathered GEMM ``g`` (float64), input planes in [B, IH, IW, C] element order."""
    x = x_pl.double().sum(0).reshape(g.B, g.IH, g.IW, g.C)
    ys, xs = torch.arange(g.OY, device=x.device) * g.sy, torch.arange(g.OX, device=x.device) * g.sx
    cols = []
    for dy, dx in zip(g.dy, g.dx):
        iy, ix = ys + dy, xs + dx
        ok = ((iy >= 0) & (iy < g.IH))[:, None] & ((ix >= 0) & (ix < g.IW))[None, :]
        cols.append(x[:, iy.clamp(0, g.IH - 1)][:, :, ix.clamp(0, g.IW - 1)] * ok[None, :, :, None])
    return torch.cat(cols, -1).reshape(g.M, -1)


def r_gemm_gather(x_pl, w_pl, geom, bias=None, relu=False, out_f32=None, out_pl=None, out_ld=None, out_c0=0, relu_mask=None,
                  n_tile=None, mask_ld=0, mask_c0=0, colsum=None):
    W = w_pl.double().sum(0)
    out_ld = W.shape[0] if out_ld is None else out_ld
    m = torch.arange(geom.M, device=W.device)
    b, y, x = m // (geom.OY * geom.OX), (m // geom.OX) % geom.OY, m % geom.OX
    opix = (b * geom.out_H + y * geom.oys + geom.oy0) * geom.out_W + x * geom.oxs + geom.ox0
    _epilogue(_gathered(x_pl, geom) @ W.t(), opix, opix, m // 128, bias, relu, out_f32, out_pl, out_ld, out_c0, relu_mask,
              mask_ld if mask_ld else out_ld, mask_c0 if mask_ld else out_c0, colsum)
    return out_f32, out_pl


def _box_rows(x, bg, R):
    """A operand of the box GEMM for merged grid rows R: [len(R), box_px, n_chunks*64], zero outside the tensor."""
    rows, W, _ = x.shape
    xs = torch.arange(bg.box_px, device=x.device)
    parts = []
    for c0, w0, r0 in bg.chunks:
        row, px = R * bg.row_step + r0, xs + w0
        ok = ((row >= 0) & (row < rows))[:, None] & ((px >= 0) & (px < W))[None, :]
        parts.append(x[row.clamp(0, rows - 1)][:, px.clamp(0, W - 1), c0:c0 + 64] * ok[..., None])
    return torch.cat(parts, -1)


def r_gemm_box(x_pl, w_pl, bg, bias=None, relu=False, out_f32=None, out_pl=None, out_ld=None, out_c0=0, relu_mask=None,
               n_tile=None, colsum=None):
    W = w_pl.double().sum(0)
    out_ld = W.shape[0] if out_ld is None else out_ld
    R = torch.arange(bg.B * bg.hp_out, device=W.device)
    b, y = R // bg.hp_out, R % bg.hp_out
    live = (y >= bg.y0) & (y <= bg.y1)
    v = _box_rows(x_pl.double().sum(0).reshape(-1, bg.W, bg.C), bg, R[live]) @ W.t()          # [rows, px, N]
    orow = (b * bg.out_H + (y - bg.y0) * bg.oys + bg.oy0)[live][:, None]
    ocol = (torch.arange(bg.box_px, device=W.device) * bg.oxs + bg.ox0)[None, :]
    mW, mx0 = (bg.mask_W, bg.mask_x0) if bg.mask_W > 0 else (bg.out_W, 0)
    f = lambda t: t.expand(v.shape[:2]).reshape(-1)
    _epilogue(v.reshape(-1, v.shape[-1]), f(orow * bg.out_W + ocol), f(orow * mW + ocol + mx0), f((R[live] // bg.box_h)[:, None]),
              bias, relu, out_f32, out_pl, out_ld, out_c0, relu_mask, out_ld, out_c0, colsum)


def r_gemm_halo(x_pl, w_pl, hg, bias=None, relu=False, out_f32=None, out_pl=None, out_ld=None, out_c0=0, relu_mask=None,
                colsum=None):
    x = x_pl.double().sum(0).reshape(-1, hg.W, 64)
    rows = x.shape[0]
    W = w_pl.double().sum(0)
    n_sub = len(hg.subs)
    out_ld = (hg.N if hg.same_cols else W.shape[0]) if out_ld is None else out_ld
    pos = torch.arange(hg.M, device=x.device)
    R, px = pos // hg.halo_w, pos % hg.halo_w + hg.halo_w0
    b, y = R // hg.hp, R % hg.hp
    mW, mx0 = (hg.mask_W, hg.mask_x0) if hg.mask_W > 0 else (hg.out_W, 0)
    cs = torch.zeros(-(-hg.M // 128) * n_sub, hg.N, device=x.device) if colsum is not None else None
    for j, sb in enumerate(hg.subs):
        live = (y >= hg.y0) & (y <= sb["y1"]) & (px >= 0) & (px <= sb["x1"])
        Rl, pl = R[live], px[live]
        parts = []
        for dr, dc in sb["shifts"]:
            r, c = Rl + dr, pl + dc
            ok = (r >= 0) & (r < rows) & (c >= 0) & (c < hg.W)
            parts.append(x[r.clamp(0, rows - 1), c.clamp(0, hg.W - 1)] * ok[:, None])
        v = torch.cat(parts, -1) @ W[j * hg.N:(j + 1) * hg.N].t()
        orow = b[live] * hg.out_H + (y[live] - hg.y0) * hg.oys + sb["oy0"]
        ocol = pl * hg.oxs + sb["ox0"]
        c0 = out_c0 + (0 if hg.same_cols else j * hg.N)
        cs_j = torch.empty_like(cs) if colsum is not None else None
        _epilogue(v, orow * hg.out_W + ocol, orow * mW + ocol + mx0, (pos[live] // 128) * n_sub + j, bias, relu, out_f32, out_pl,
                  out_ld, c0, relu_mask, out_ld, c0, cs_j)
        if colsum is not None:
            cs += cs_j                                                       # sub-item j owns rows (tile, j) only
    if colsum is not None:
        colsum.view(-1, hg.N).copy_(cs)


def _split_rows(M, splits, unit):
    per = -(-(-(-M // splits)) // unit) * unit
    return [(s * per, min(M, (s + 1) * per)) for s in range(splits)]


def r_wgrad_gather(x_pl, g_pl, geom, splits, n_tile=None):
    A = _gathered(x_pl, geom)
    G = g_pl.double().sum(0).reshape(geom.M, -1)
    return torch.stack([(A[lo:hi].t() @ G[lo:hi]).float() for lo, hi in _split_rows(geom.M, splits, tc.KC)])


def r_wgrad_box(x_pl, g_pl, bg, box_h, splits):
    g = g_pl.double().sum(0)                                              # [g_rows, sites per row, N]
    A = _box_rows(x_pl.double().sum(0).reshape(-1, bg.W, bg.C), bg, torch.arange(g.shape[0]))
    return torch.stack([torch.einsum("rpk,rpn->kn", A[lo:hi], g[lo:hi]).float() for lo, hi in _split_rows(g.shape[0], splits, box_h)])


def r_wgrad_reduce(partials, N, C, KH, KW, out=None, accumulate=False, scale=1.0):
    s = partials.double().sum(0).float() * np.float32(scale)             # [(kh, kw, c), N]
    dw = s.t().reshape(N, KH, KW, C).permute(0, 3, 1, 2)
    if out is None:
        return dw.contiguous()
    o = out.view(N, C, KH, KW)                                        # the kernel writes the memory of any contiguous shape
    if accumulate:
        o += dw
    else:
        o.copy_(dw)
    return out


def r_bias_grad(colsum, N, out=None, accumulate=False):
    return r_wgrad_reduce(colsum.view(-1, 1, N), N, 1, 1, 1, out=out, accumulate=accumulate).view(N)


@pytest.fixture
def host_k12(monkeypatch):
    """tc_conv's launch wrappers replaced by the restatements above (the encoder classes look them up at call time)."""
    for name, fn in (("split_bf16", r_split_bf16), ("pack_weights", r_pack_weights), ("pack_conv_weight", r_pack_conv_weight), ("gemm_gather", r_gemm_gather),
                     ("gemm_box", r_gemm_box), ("gemm_halo", r_gemm_halo), ("wgrad_gather", r_wgrad_gather),
                     ("wgrad_box", r_wgrad_box), ("wgrad_reduce", r_wgrad_reduce), ("bias_grad", r_bias_grad)):
        monkeypatch.setattr(tc, name, fn)
    return monkeypatch


def _encoder_modules(fc_out=512, seed=0):
    """AC_CNN_Atari's encoder (orthogonal, gain sqrt 2) with seeded non-zero biases, so that every bias reaches a check."""
    import torch.nn as nn
    torch.manual_seed(seed)
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    fc = nn.Linear(6400, fc_out) if fc_out else None
    for m in convs + ([fc] if fc is not None else []):
        nn.init.orthogonal_(m.weight, gain=np.sqrt(2))
        nn.init.uniform_(m.bias, -0.1, 0.1)
    return convs, fc


def _run(enc, x_pl, B, dz):
    for p in enc.parameters():
        p.grad = None
    z = tc.tc_encode(enc, x_pl, B)
    z.backward(dz)
    return z.detach(), [p.grad.clone() for p in enc.parameters()]


@pytest.mark.parametrize("box_wgrad", ["", "2", "3", "23"])
@pytest.mark.parametrize("halo", ["0", "2", "3"])
def test_box_encoder_orchestration_against_float64(host_k12, halo, box_wgrad):
    """BoxNatureCNN.forward / .backward at B = 2 on the restated launches, every XB_K12_HALO / XB_K12_BOX_WGRAD path: each
    layer and gradient against float64 from the encoder's own stored inputs, the padding of the persistent buffers bitwise
    zero after one and after a second forward / backward on other data, and gradients added into existing ``.grad``
    tensors (the flat-bucket optimizer's layout) equal to ``prev + fresh`` bit for bit."""
    import k12_encoder_refs as K
    host_k12.setattr(tc, "HALO", halo != "0")
    host_k12.setattr(tc, "HALO3", halo == "3")
    host_k12.setattr(tc, "BOX_WGRAD2", "2" in box_wgrad)
    host_k12.setattr(tc, "BOX_WGRAD3", "3" in box_wgrad)
    B = 2
    convs, fc = _encoder_modules()
    enc = tc.BoxNatureCNN(convs, fc, (84, 84, 4), backend=tc.CudaBackend(3))
    gen = torch.Generator().manual_seed(1)
    obs = [torch.randint(0, 256, (B, 84, 84, 4), generator=gen, dtype=torch.uint8) for _ in range(2)]
    dzs = [torch.randn(B, 512, generator=gen) for _ in range(2)]
    for i in (0, 1):
        x_pl = r_split_bf16(obs[i].float(), 1)                     # the raw uint8 pixels as one exact plane
        z, grads = _run(enc, x_pl, B, dzs[i])
        K.check_padding(enc, B)
        ratios = K.check(enc, K.capture(enc, B, x_pl, z, grads), dzs[i])
        assert set(ratios) >= {"act1", "act2", "act3", "z", "y", "g3", "g2", "g1", "fc.weight", "conv1.bias"}
    # accumulation into existing .grad
    prev = [torch.randn(p.shape, generator=gen) for p in enc.parameters()]
    for p, g in zip(enc.parameters(), prev):
        p.grad = g.clone()
    tc.tc_encode(enc, x_pl, B).backward(dzs[1])
    for i, (p, g, f) in enumerate(zip(enc.parameters(), prev, grads)):
        assert torch.equal(p.grad, g + f), "parameter %d: .grad is not prev + fresh" % i


@pytest.mark.parametrize("fc_out", [512, 0])
def test_gathered_encoder_orchestration_against_float64(host_k12, fc_out):
    """TensorCoreNatureCNN (the XB_K12_BOX=0 path) and the Basic_CNN shape (no hidden layer) through the same checker, the
    data gradients recovered by the recording backend."""
    import k12_encoder_refs as K
    B = 2
    convs, fc = _encoder_modules(fc_out, seed=1)
    gen = torch.Generator().manual_seed(2)
    obs = torch.randint(0, 256, (B, 84, 84, 4), generator=gen, dtype=torch.uint8)
    x_pl = r_split_bf16(obs.float() / 255.0, 3)
    for cls in (tc.TensorCoreNatureCNN, tc.BoxNatureCNN):
        enc = cls(convs, fc, (84, 84, 4), backend=K.RecordingBackend(3))
        dz = torch.randn(B, fc_out, generator=gen) if fc_out else torch.randn(B * 100, 64, generator=gen)
        z, grads = _run(enc, x_pl, B, dz)
        K.check(enc, K.capture(enc, B, x_pl, z, grads), dz)

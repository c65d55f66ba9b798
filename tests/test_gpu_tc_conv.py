"""GPU parity tests of the K12 tensor-core layers (xuance_b200/csrc/conv_tc.cu) against float64 references: operand
preparation, forward (2 / 3 planes, raw uint8 single plane), data gradient with a given ReLU mask, weight gradient
(MN-major operands, site splits, column tiles), the Linear layer in all three modes, the whole encoder forward + backward
next to cuDNN fp32, and a PPO update with compute="tc" next to the fp32 learner.

Tolerances.  Operands with 3 planes are exact to 2^-24; what remains is the float32 accumulation of the tensor core, which
truncates on every addition of a 16-deep product block (results are biased toward zero by up to ~0.5 ulp per K step of
the hi.hi accumulator).  For O(1) outputs of K <= 576 layers that is <= 3e-6; the 6400-deep Linear and the long site
reductions of the weight gradients carry proportionally more and are bounded by cutting the reduction (wgrad_splits)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _planes_ref(x, planes):
    r, out = x.clone(), []
    for _ in range(planes):
        h = r.bfloat16()
        out.append(h)
        r = r - h.float()
    return torch.stack(out)


@pytest.mark.parametrize("planes", [1, 2, 3])
def test_split_and_pack(planes):
    from xuance_b200.torch.utils import tc_conv as tc
    for shape in ((1000, 37), (4099,), (8, 8)):                      # 37000 = 8*4625, a ragged length, one vector
        x = torch.randn(*shape, device=DEV)
        assert torch.equal(tc.split_bf16(x, planes), _planes_ref(x, planes))
    w = torch.randn(32, 4, 8, 8, device=DEV)
    assert torch.equal(tc.pack_conv_weight(w, planes), _planes_ref(w.permute(0, 2, 3, 1).reshape(32, -1), planes))
    s = np.float32(1.0 / 255.0)
    assert torch.equal(tc.pack_conv_weight(w, planes, 1.0 / 255.0),
                       _planes_ref((w.permute(0, 2, 3, 1).reshape(32, -1).cpu() * s).to(DEV), planes))


def _forward_conv(B, H, W, C, N, k, s, planes, atol):
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(0)
    pad = (k - s) // 2
    x = torch.rand(B, H, W, C, device=DEV)
    w = torch.randn(N, C, k, k, device=DEV) / np.sqrt(C * k * k)
    b = torch.randn(N, device=DEV) * 0.1
    g = tc.conv_forward_geometry(B, H, W, C, k, k, s, pad)
    out = torch.full((g.M, N), float("nan"), device=DEV)
    opl = torch.zeros((planes, g.M, N), dtype=torch.bfloat16, device=DEV)
    tc.gemm_gather(tc.split_bf16(x, planes), tc.pack_conv_weight(w, planes), g, bias=b, relu=True, out_f32=out, out_pl=opl)
    want = F.relu(F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), stride=s, padding=pad))
    want = want.permute(0, 2, 3, 1).reshape(g.M, N)
    np.testing.assert_allclose(out.cpu().numpy(), want.cpu().numpy(), rtol=0, atol=atol)
    assert torch.equal(opl, _planes_ref(out, planes))               # the planes are the split of the float32 result


LAYERS = [(2, 84, 84, 4, 32, 8, 4), (3, 21, 21, 32, 64, 4, 2), (5, 10, 10, 64, 64, 3, 1), (256, 21, 21, 32, 64, 4, 2)]
if os.environ.get("XB_SANITIZE") == "1":       # under compute-sanitizer, which slows kernels 10-100x
    LAYERS = LAYERS[:3]


@pytest.mark.parametrize("B,H,W,C,N,k,s", LAYERS)
def test_forward_conv_two_planes(B, H, W, C, N, k, s):
    _forward_conv(B, H, W, C, N, k, s, 2, 5e-5)


@pytest.mark.parametrize("B,H,W,C,N,k,s", LAYERS)
def test_forward_conv_three_planes(B, H, W, C, N, k, s):
    """Three planes (hi, mid, lo), six products in three accumulators: float32-grade."""
    _forward_conv(B, H, W, C, N, k, s, 3, 3e-6)


@pytest.mark.parametrize("planes", [2, 3])
def test_forward_conv1_raw_uint8_plane(planes):
    """conv1 fed with ONE exact bf16 plane of raw pixel values; the packed weights carry 1/255 (cnn.py:98 folded)."""
    from xuance_b200 import _lib
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(1)
    B, H, W, C, N, k, s = 9, 84, 84, 4, 32, 8, 4
    obs = torch.randint(0, 256, (B, H, W, C), dtype=torch.uint8, device=DEV)
    w = torch.randn(N, C, k, k, device=DEV) / np.sqrt(C * k * k)
    b = torch.randn(N, device=DEV) * 0.1
    raw = torch.empty((1, B, H, W, C), dtype=torch.bfloat16, device=DEV)
    _lib.call("xb_gather_obs_planes", _lib.ptr(obs), None, B, H * W * C, 1, _lib.ptr(raw))
    assert torch.equal(raw[0].float(), obs.float())
    g = tc.conv_forward_geometry(B, H, W, C, k, k, s, 2)
    out = torch.full((g.M, N), float("nan"), device=DEV)
    tc.gemm_gather(raw, tc.pack_conv_weight(w, planes, 1.0 / 255.0), g, bias=b, relu=True, out_f32=out)
    want = F.relu(F.conv2d((obs.double() / 255.0).permute(0, 3, 1, 2), w.double(), b.double(), stride=s, padding=2))
    np.testing.assert_allclose(out.cpu().numpy(), want.permute(0, 2, 3, 1).reshape(g.M, N).cpu().numpy(), rtol=0,
                               atol=5e-5 if planes == 2 else 3e-6)


@pytest.mark.parametrize("planes,atol", [(2, 5e-5), (3, 3e-6)])
@pytest.mark.parametrize("B,H,W,C,N,k,s", [(3, 21, 21, 32, 64, 4, 2), (5, 10, 10, 64, 64, 3, 1), (64, 21, 21, 32, 64, 4, 2)])
def test_data_gradient_with_mask(B, H, W, C, N, k, s, planes, atol):
    """grad_input of one convolution (one GEMM per stride phase) times a GIVEN ReLU-derivative mask vs autograd."""
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(1)
    pad = (k - s) // 2
    x = torch.randn(B, C, H, W, device=DEV, dtype=torch.float64, requires_grad=True)
    w = torch.randn(N, C, k, k, device=DEV) / np.sqrt(N * k * k / (s * s))
    y = F.conv2d(x, w.double(), stride=s, padding=pad)
    gy = torch.randn(y.shape, device=DEV)
    (want,) = torch.autograd.grad(y, x, gy.double())
    act = torch.randn(B, H, W, C, device=DEV)                      # the "saved activation": mask = act > 0
    act_hi = act.bfloat16()
    want = want.permute(0, 2, 3, 1) * (act_hi.float() > 0)
    g_pl = tc.split_bf16(gy.permute(0, 2, 3, 1).reshape(-1, N).contiguous(), planes)
    opl = torch.full((planes, B * H * W, C), float("nan"), dtype=torch.bfloat16, device=DEV)
    for geom, taps in tc.conv_dgrad_geometries(B, H, W, C, k, k, s, pad, N):
        tc.gemm_gather(g_pl, tc.split_bf16(tc.dgrad_weight_matrix(w, taps), planes), geom, out_pl=opl, out_ld=C, relu_mask=act_hi)
    got = opl.float().sum(0).reshape(B, H, W, C)
    np.testing.assert_allclose(got.cpu().numpy(), want.cpu().numpy(), rtol=0, atol=atol)


@pytest.mark.parametrize("B,H,W,C,N,k,s", [(2, 84, 84, 4, 32, 8, 4), (4, 21, 21, 32, 64, 4, 2), (5, 10, 10, 64, 64, 3, 1),
                                            (64, 84, 84, 4, 32, 8, 4), (256, 10, 10, 64, 64, 3, 1)])
def test_weight_gradient(B, H, W, C, N, k, s):
    """grad_weight of one convolution (MN-major operands, site splits, ordered reduce) vs autograd in float64.  The bound
    grows with the K steps one accumulator chain spans (truncating additions); wgrad_splits keeps chains <= 4096 sites."""
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(2)
    pad = (k - s) // 2
    x = torch.rand(B, H, W, C, device=DEV)
    w = (torch.randn(N, C, k, k, device=DEV, dtype=torch.float64) / np.sqrt(C * k * k)).requires_grad_(True)
    y = F.conv2d(x.permute(0, 3, 1, 2).double(), w, stride=s, padding=pad)
    gy = torch.randn(y.shape, device=DEV) / np.sqrt(y[0, 0].numel() * B)
    (want,) = torch.autograd.grad(y, w, gy.double())
    g = tc.conv_forward_geometry(B, H, W, C, k, k, s, pad)
    scale = float(want.abs().max())
    for planes, base in ((2, 5e-5), (3, 2e-6)):
        x_pl = tc.split_bf16(x, planes)
        g_pl = tc.split_bf16(gy.permute(0, 2, 3, 1).reshape(g.M, N).contiguous(), planes)
        for splits in sorted({1, tc.wgrad_splits(g.M, g.K)}):
            steps = -(-g.M // splits) / 16.0
            dw = tc.wgrad_reduce(tc.wgrad_gather(x_pl, g_pl, g, splits), N, C, k, k)
            np.testing.assert_allclose(dw.cpu().numpy(), want.cpu().numpy(), rtol=0,
                                       atol=max(base, 1.2e-7 * steps) * max(scale, 1.0),
                                       err_msg="planes=%d splits=%d" % (planes, splits))


def test_weight_gradient_raw_uint8_plane():
    """conv1's weight gradient from ONE raw pixel plane and three gradient planes; the reduce carries the 1/255."""
    from xuance_b200 import _lib
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(3)
    B, H, W, C, N, k, s = 16, 84, 84, 4, 32, 8, 4
    obs = torch.randint(0, 256, (B, H, W, C), dtype=torch.uint8, device=DEV)
    w = (torch.randn(N, C, k, k, device=DEV, dtype=torch.float64) / 16).requires_grad_(True)
    y = F.conv2d((obs.double() / 255.0).permute(0, 3, 1, 2), w, stride=s, padding=2)
    gy = torch.randn(y.shape, device=DEV) / np.sqrt(441 * B)
    (want,) = torch.autograd.grad(y, w, gy.double())
    raw = torch.empty((1, B, H, W, C), dtype=torch.bfloat16, device=DEV)
    _lib.call("xb_gather_obs_planes", _lib.ptr(obs), None, B, H * W * C, 1, _lib.ptr(raw))
    g = tc.conv_forward_geometry(B, H, W, C, k, k, s, 2)
    g_pl = tc.split_bf16(gy.permute(0, 2, 3, 1).reshape(g.M, N).contiguous(), 3)
    dw = tc.wgrad_reduce(tc.wgrad_gather(raw, g_pl, g, tc.wgrad_splits(g.M, g.K)), N, C, k, k, scale=1.0 / 255.0)
    np.testing.assert_allclose(dw.cpu().numpy(), want.cpu().numpy(), rtol=0, atol=3e-6 * max(1.0, float(want.abs().max())))


@pytest.mark.parametrize("planes,atol", [(2, 1e-4), (3, 2e-5)])
def test_linear_layer_all_modes(planes, atol):
    """Linear(6400 -> 512) forward (column tiles inside one launch), its data gradient (6400 columns = 50 / 100 column
    tiles) and its weight gradient (column tiles of a gradient matrix with 512 elements per row, site splits)."""
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(4)
    B, K, N = 300, 6400, 512
    x = torch.rand(B, K, device=DEV)
    w = torch.randn(N, K, device=DEV, dtype=torch.float64) / 80.0
    b = torch.randn(N, device=DEV) * 0.1
    x_pl = tc.split_bf16(x, planes)
    w_pl = tc.split_bf16(w.float(), planes)
    out = torch.full((B, N), float("nan"), device=DEV)
    tc.gemm_gather(x_pl, w_pl, tc.linear_geometry(B, K), bias=b, relu=True, out_f32=out)
    want = F.relu(x.double() @ w.float().double().t() + b.double())
    np.testing.assert_allclose(out.cpu().numpy(), want.cpu().numpy(), rtol=0, atol=atol)
    gy = torch.randn(B, N, device=DEV) / 16
    g_pl = tc.split_bf16(gy, planes)
    wt_pl = tc.split_bf16(w.float().t().contiguous(), planes)        # [K, N]: rows = output columns of the data gradient
    dx = torch.full((B, K), float("nan"), device=DEV)
    tc.gemm_gather(g_pl, wt_pl, tc.linear_geometry(B, N), out_f32=dx)
    np.testing.assert_allclose(dx.cpu().numpy(), (gy.double() @ w.float().double()).cpu().numpy(), rtol=0, atol=atol)
    geom = tc.linear_geometry(B, K)
    nt = N // tc.n_tile_for(N, planes)
    dw = tc.wgrad_reduce(tc.wgrad_gather(x_pl, g_pl, geom, tc.wgrad_splits(B, K, nt)), N, K, 1, 1).reshape(N, K)
    np.testing.assert_allclose(dw.cpu().numpy(), (gy.double().t() @ x.double()).cpu().numpy(), rtol=0, atol=atol)


@pytest.mark.parametrize("planes,atol", [(2, 5e-5), (3, 3e-6)])
def test_box_convolutions_forward_and_data_gradient(planes, atol):
    """conv2 / conv3 forward and their data gradients with the A operand fetched by TMA boxes from padded-row activations
    (xb_gemm_box_tc): every geometry BoxNatureCNN builds, against float64 convolutions / autograd."""
    import torch.nn as nn
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(11)
    B = 5
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    enc = tc.BoxNatureCNN([c.to(DEV) for c in convs], None, (84, 84, 4), backend=tc.CudaBackend(planes))
    P = enc._plan(B)
    hp1, hp2, off1 = P["hp1"], P["hp2"], P["off1"]
    a1 = torch.rand(B, 21, 21, 32, device=DEV)                               # conv2's input (conv1's activation)
    W1p, xo1 = P["W1p"], P["xo1"]                                            # one zero pixel on the left: pixel pairs are 128 B
    assert (W1p, xo1) == (22, 1)
    act1 = torch.zeros(planes, B, hp1, W1p, 32, dtype=torch.bfloat16, device=DEV)
    act1[:, :, off1:off1 + 21, xo1:xo1 + 21] = tc.split_bf16(a1, planes)
    act1 = act1.view(planes, B * hp1, W1p, 32)
    act1_pairs = act1.view(planes, B * hp1, W1p // 2, 64)
    w2, b2 = convs[1].weight.detach(), convs[1].bias.detach()
    out2 = torch.zeros(planes, B * hp2, 10, 64, dtype=torch.bfloat16, device=DEV)
    tc.gemm_box(act1_pairs, tc.pack_conv_weight(w2, planes), P["fwd2"], bias=b2, relu=True, out_pl=out2, out_ld=64)
    want2 = F.relu(F.conv2d(a1.permute(0, 3, 1, 2).double(), w2.double(), b2.double(), stride=2, padding=1)).permute(0, 2, 3, 1)
    got2 = out2.float().sum(0).view(B, hp2, 10, 64)
    np.testing.assert_allclose(got2[:, 1:11].cpu().numpy(), want2.cpu().numpy(), rtol=0, atol=atol)
    assert float(got2[:, 0].abs().max()) == 0.0 and float(got2[:, 11].abs().max()) == 0.0      # padding rows never written
    # conv3 forward from the padded act2 into the plain matrix
    w3, b3 = convs[2].weight.detach(), convs[2].bias.detach()
    a2 = got2[:, 1:11].contiguous()
    out3 = torch.full((B * 100, 64), float("nan"), device=DEV)
    tc.gemm_box(out2, tc.pack_conv_weight(w3, planes), P["fwd3"], bias=b3, relu=True, out_f32=out3, out_ld=64)
    want3 = F.relu(F.conv2d(a2.permute(0, 3, 1, 2).double(), w3.double(), b3.double(), stride=1, padding=1)).permute(0, 2, 3, 1)
    np.testing.assert_allclose(out3.view(B, 10, 10, 64).cpu().numpy(), want3.cpu().numpy(), rtol=0, atol=atol)
    # conv3 data gradient (mask = act2 plane 0) into act2's padded layout
    g3 = torch.randn(B, 10, 10, 64, device=DEV)
    g3p = torch.zeros(planes, B, hp2, 10, 64, dtype=torch.bfloat16, device=DEV)
    g3p[:, :, 1:11] = tc.split_bf16(g3, planes)
    g3p = g3p.view(planes, B * hp2, 10, 64)
    x2 = a2.double().permute(0, 3, 1, 2).requires_grad_(True)
    y3 = F.conv2d(x2, w3.double(), stride=1, padding=1)
    (dx2,) = torch.autograd.grad(y3, x2, g3.double().permute(0, 3, 1, 2))
    want = dx2.permute(0, 2, 3, 1) * (out2[0].float().view(B, hp2, 10, 64)[:, 1:11] > 0)
    d2 = torch.zeros(planes, B * hp2, 10, 64, dtype=torch.bfloat16, device=DEV)
    cs2 = torch.full((P["dg3"].m_tiles, 64), float("nan"), device=DEV)
    tc.gemm_box(g3p, tc.split_bf16(tc.dgrad_weight_matrix(w3, P["taps3"]), planes), P["dg3"], out_pl=d2, out_ld=64, relu_mask=out2[0],
                colsum=cs2)
    np.testing.assert_allclose(d2.float().sum(0).view(B, hp2, 10, 64)[:, 1:11].cpu().numpy(), want.cpu().numpy(), rtol=0, atol=atol * 4)
    # fused bias-gradient partials: column sums of exactly the rows written (padding / garbage rows contribute nothing)
    np.testing.assert_allclose(tc.bias_grad(cs2, 64).cpu().numpy(), want.sum((0, 1, 2)).cpu().numpy(), rtol=0, atol=atol * 400)
    # conv2 data gradient: four stride phases into act1's padded layout (mask = act1 plane 0)
    g2 = torch.randn(B, 10, 10, 64, device=DEV)
    g2p = torch.zeros(planes, B, hp2, 10, 64, dtype=torch.bfloat16, device=DEV)
    g2p[:, :, 1:11] = tc.split_bf16(g2, planes)
    g2p = g2p.view(planes, B * hp2, 10, 64)
    x1 = a1.double().permute(0, 3, 1, 2).requires_grad_(True)
    y2 = F.conv2d(x1, w2.double(), stride=2, padding=1)
    (dx1,) = torch.autograd.grad(y2, x1, g2.double().permute(0, 3, 1, 2))
    mask1 = act1[0].float().view(B, hp1, W1p, 32)[:, off1:off1 + 21, xo1:xo1 + 21] > 0
    d1 = torch.zeros(planes, B * hp1, 21, 32, dtype=torch.bfloat16, device=DEV)
    cs1 = torch.full((sum(bg.m_tiles for bg, _ in P["dg2"]), 32), float("nan"), device=DEV)
    row = 0
    for bg, taps in P["dg2"]:
        tc.gemm_box(g2p, tc.split_bf16(tc.dgrad_weight_matrix(w2, taps), planes), bg, out_pl=d1, out_ld=32, relu_mask=act1[0],
                    colsum=cs1[row:row + bg.m_tiles])
        row += bg.m_tiles
    got1 = d1.float().sum(0).view(B, hp1, 21, 32)
    np.testing.assert_allclose(tc.bias_grad(cs1, 32).cpu().numpy(), (dx1.permute(0, 2, 3, 1) * mask1).sum((0, 1, 2)).cpu().numpy(),
                               rtol=0, atol=atol * 2000)
    np.testing.assert_allclose(got1[:, off1:off1 + 21].cpu().numpy(), (dx1.permute(0, 2, 3, 1) * mask1).cpu().numpy(), rtol=0, atol=atol * 4)
    assert float(got1[:, :off1].abs().max()) == 0.0
    # weight gradients of conv3 and conv2 with both operands as TMA boxes (reduction chunks of 6 grid rows = 60 sites)
    for w, x_pad, g_pad, bg, xin, gout, stride, cin in ((w3, out2, g3p, P["fwd3"], a2, g3, 1, 64), (w2, act1_pairs, g2p, P["fwd2"], a1, g2, 2, 32)):
        wd = w.double().requires_grad_(True)
        y = F.conv2d(xin.double().permute(0, 3, 1, 2), wd, stride=stride, padding=1)
        (want_w,) = torch.autograd.grad(y, wd, gout.double().permute(0, 3, 1, 2))
        k = w.shape[-1]
        for splits in (1, 3):
            dw = tc.wgrad_reduce(tc.wgrad_box(x_pad, g_pad.view(planes, B * hp2, 10, 64), bg, 6, splits), 64, cin, k, k)
            np.testing.assert_allclose(dw.cpu().numpy(), want_w.cpu().numpy(), rtol=0, atol=atol * 8 * max(1.0, float(want_w.abs().max())),
                                       err_msg="cin=%d splits=%d" % (cin, splits))
        # the same gradients through the gathered kernel over the padded tensors (BoxNatureCNN's default for conv2)
        geo = P["wg3"] if cin == 64 else P["wg2"]
        x_plain = x_pad if cin == 64 else act1
        dw = enc.be.wgrad(x_plain, g_pad.view(planes, -1, 64), geo, 64, cin, k, k)
        np.testing.assert_allclose(dw.cpu().numpy(), want_w.cpu().numpy(), rtol=0, atol=atol * 8 * max(1.0, float(want_w.abs().max())),
                                   err_msg="gathered over padded rows, cin=%d" % cin)


def test_pack_weights_one_launch_equals_the_single_form_launches():
    """xb_pack_weights: forward pack, transposed pack and data-gradient matrices of several weights in one launch are bit-equal
    to xb_pack_conv_weight / transpose + xb_split_bf16 / dgrad_weight_matrix + xb_split_bf16."""
    from xuance_b200 import _lib
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(2)
    w2 = torch.randn(64, 32, 4, 4, device=DEV)
    w3 = torch.randn(64, 64, 3, 3, device=DEV)
    w4 = torch.randn(48, 64, 5, 5, device=DEV)
    taps3 = [(kh, kw) for kh in range(3) for kw in range(3)]
    taps2 = [(1, 0), (1, 2), (3, 0), (3, 2)]
    for planes in (2, 3):
        outs = tc.pack_weights([(w2, _lib.PACK_FORWARD, None, 1.0 / 255.0), (w3, _lib.PACK_DGRAD, taps3, 1.0),
                                (w2, _lib.PACK_DGRAD, taps2, 1.0), (w4, _lib.PACK_FORWARD, None, 1.0),
                                (w4, _lib.PACK_TRANSPOSED, None, 1.0)], planes, DEV)
        want = [tc.pack_conv_weight(w2, planes, 1.0 / 255.0), tc.split_bf16(tc.dgrad_weight_matrix(w3, taps3), planes),
                tc.split_bf16(tc.dgrad_weight_matrix(w2, taps2), planes), tc.pack_conv_weight(w4, planes),
                tc.split_bf16(w4.permute(0, 2, 3, 1).reshape(48, 1600).t().contiguous(), planes)]
        for i, (a, b) in enumerate(zip(outs, want)):
            assert a.shape == b.shape, (i, a.shape, b.shape)
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "form %d planes %d" % (i, planes)
    # many taps (a Linear layer over a [C, H, W] feature map): the shared-memory tiled transposes of pack and reduce
    w5 = torch.randn(64, 32, 10, 10, device=DEV)
    f, t = tc.pack_weights([(w5, _lib.PACK_FORWARD, None, 1.0), (w5, _lib.PACK_TRANSPOSED, None, 0.5)], 3, DEV)
    kmaj = w5.permute(0, 2, 3, 1).reshape(64, 3200)
    assert torch.equal(f.view(torch.int16), tc.split_bf16(kmaj.contiguous(), 3).view(torch.int16))
    assert torch.equal(t.view(torch.int16), tc.split_bf16((kmaj * 0.5).t().contiguous(), 3).view(torch.int16))
    part = torch.randn(3, 3200, 64, device=DEV)
    want_dw = (part.double().sum(0) * 0.25).t().reshape(64, 10, 10, 32).permute(0, 3, 1, 2)
    dw = tc.wgrad_reduce(part.clone(), 64, 32, 10, 10, scale=0.25)
    np.testing.assert_allclose(dw.cpu().numpy(), want_dw.cpu().numpy(), rtol=0, atol=2e-6)
    acc = torch.ones(64, 32, 10, 10, device=DEV)
    tc.wgrad_reduce(part.clone(), 64, 32, 10, 10, out=acc, accumulate=True, scale=0.25)
    np.testing.assert_allclose(acc.cpu().numpy(), want_dw.cpu().numpy() + 1.0, rtol=0, atol=2e-6)


@pytest.mark.parametrize("planes,atol", [(2, 5e-5), (3, 3e-6)])
def test_linear_data_gradient_into_padded_rows_with_mask_and_colsum(planes, atol):
    """The Linear layer's data gradient written at a column offset of wider rows (conv3's padded output-gradient tensor), with
    the ReLU mask read from a plain matrix (mask_ld / mask_c0) and the fused column sums (bias-gradient partials)."""
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(5)
    B, N_in, N_out, ld, c0 = 300, 128, 640, 768, 64
    g = torch.randn(B, N_in, device=DEV)
    w = torch.randn(N_in, N_out, device=DEV) / 8          # [K, N] of the data-gradient GEMM
    act = torch.randn(B, N_out, device=DEV)
    mask_pl = tc.split_bf16(act, planes)
    out = torch.zeros(planes, B, ld, dtype=torch.bfloat16, device=DEV)
    cs = torch.full((-(-B // 128), N_out), float("nan"), device=DEV)
    tc.gemm_gather(tc.split_bf16(g, planes), tc.split_bf16(w.t().contiguous(), planes), tc.linear_geometry(B, N_in), out_pl=out,
                   out_ld=ld, out_c0=c0, relu_mask=mask_pl[0], mask_ld=N_out, mask_c0=0, colsum=cs)
    want = (g.double() @ w.double()) * (mask_pl[0].float() > 0)
    got = out.float().sum(0)
    np.testing.assert_allclose(got[:, c0:c0 + N_out].cpu().numpy(), want.cpu().numpy(), rtol=0, atol=atol * 8)
    assert float(got[:, :c0].abs().max()) == 0.0 and float(got[:, c0 + N_out:].abs().max()) == 0.0
    np.testing.assert_allclose(cs.sum(0).cpu().numpy(), want.sum(0).cpu().numpy(), rtol=0, atol=atol * 800)
    np.testing.assert_allclose(tc.bias_grad(cs, 64).cpu().numpy(), want.view(B, 10, 64).sum((0, 1)).cpu().numpy(), rtol=0, atol=atol * 8000)


@pytest.mark.parametrize("planes,atol", [(2, 5e-5), (3, 3e-6)])
def test_halo_convolutions_forward_and_data_gradients(planes, atol):
    """xb_gemm_halo_tc (activation tile resident in shared memory, taps = descriptor offsets into it): conv3 forward, its data
    gradient, and the four stride phases of conv2's data gradient in ONE launch - against float64 convolutions / autograd, with
    masks, fused column sums and the padded / strided output placements BoxNatureCNN uses.  B = 37 images: 37 * 144 raster
    positions are not a multiple of the 128-position M tile, and tiles straddle image boundaries."""
    import torch.nn as nn
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(13)
    B = 37
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    enc = tc.BoxNatureCNN([c.to(DEV) for c in convs], None, (84, 84, 4), backend=tc.CudaBackend(planes))
    P = enc._plan(B)
    hp1, hp2, off1, W1p, xo1 = P["hp1"], P["hp2"], P["off1"], P["W1p"], P["xo1"]
    w2, w3, b3 = convs[1].weight.detach(), convs[2].weight.detach(), convs[2].bias.detach()
    pad2 = lambda t: torch.cat([torch.zeros_like(t[:, :, :1]), t, torch.zeros_like(t[:, :, :1])], 2).reshape(planes, B * hp2, 10, 64)
    # conv3 forward from the padded act2
    a2 = torch.rand(B, 10, 10, 64, device=DEV)
    act2 = pad2(tc.split_bf16(a2, planes))
    out3 = torch.full((B * 100, 64), float("nan"), device=DEV)
    act3 = torch.zeros(planes, B * 100, 64, dtype=torch.bfloat16, device=DEV)
    tc.gemm_halo(act2, tc.pack_conv_weight(w3, planes), P["h_fwd3"], bias=b3, relu=True, out_f32=out3, out_pl=act3, out_ld=64)
    want3 = F.relu(F.conv2d(a2.permute(0, 3, 1, 2).double(), w3.double(), b3.double(), stride=1, padding=1)).permute(0, 2, 3, 1)
    np.testing.assert_allclose(out3.view(B, 10, 10, 64).cpu().numpy(), want3.cpu().numpy(), rtol=0, atol=atol)
    np.testing.assert_allclose(act3.float().sum(0).view(B, 10, 10, 64).cpu().numpy(), want3.cpu().numpy(), rtol=0, atol=atol)
    # conv3 data gradient into act2's padded layout, mask = act2 plane 0, column sums
    g3 = torch.randn(B, 10, 10, 64, device=DEV)
    g3p = pad2(tc.split_bf16(g3, planes))
    x2 = a2.double().permute(0, 3, 1, 2).requires_grad_(True)
    (dx2,) = torch.autograd.grad(F.conv2d(x2, w3.double(), stride=1, padding=1), x2, g3.double().permute(0, 3, 1, 2))
    want = dx2.permute(0, 2, 3, 1) * (act2[0].float().view(B, hp2, 10, 64)[:, 1:11] > 0)
    d2 = torch.zeros(planes, B * hp2, 10, 64, dtype=torch.bfloat16, device=DEV)
    cs2 = torch.full((P["h_dg3"].m_tiles, 64), float("nan"), device=DEV)
    tc.gemm_halo(g3p, tc.split_bf16(tc.dgrad_weight_matrix(w3, P["taps3"]), planes), P["h_dg3"], out_pl=d2, out_ld=64,
                 relu_mask=act2[0], colsum=cs2)
    got2 = d2.float().sum(0).view(B, hp2, 10, 64)
    np.testing.assert_allclose(got2[:, 1:11].cpu().numpy(), want.cpu().numpy(), rtol=0, atol=atol * 4)
    assert float(got2[:, 0].abs().max()) == 0.0 and float(got2[:, 11].abs().max()) == 0.0
    np.testing.assert_allclose(tc.bias_grad(cs2, 64).cpu().numpy(), want.sum((0, 1, 2)).cpu().numpy(), rtol=0, atol=atol * 3000)
    # conv2 data gradient: the four stride phases as the sub-items of one launch, into act1's padded layout (mask: act1 plane 0)
    a1 = torch.rand(B, 21, 21, 32, device=DEV) - 0.3
    act1 = torch.zeros(planes, B, hp1, W1p, 32, dtype=torch.bfloat16, device=DEV)
    act1[:, :, off1:off1 + 21, xo1:xo1 + 21] = tc.split_bf16(a1, planes)
    act1 = act1.view(planes, B * hp1, W1p, 32)
    g2 = torch.randn(B, 10, 10, 64, device=DEV)
    g2p = pad2(tc.split_bf16(g2, planes))
    x1 = a1.double().permute(0, 3, 1, 2).requires_grad_(True)
    (dx1,) = torch.autograd.grad(F.conv2d(x1, w2.double(), stride=2, padding=1), x1, g2.double().permute(0, 3, 1, 2))
    mask1 = act1[0].float().view(B, hp1, W1p, 32)[:, off1:off1 + 21, xo1:xo1 + 21] > 0
    want1 = dx1.permute(0, 2, 3, 1) * mask1
    d1 = torch.zeros(planes, B * hp1, 21, 32, dtype=torch.bfloat16, device=DEV)
    wd2 = torch.cat([tc.split_bf16(tc.dgrad_weight_matrix(w2, taps), planes) for _, taps in P["dg2"]], 1).contiguous()
    cs1 = torch.full((P["h_dg2"].m_tiles, 32), float("nan"), device=DEV)
    tc.gemm_halo(g2p, wd2, P["h_dg2"], out_pl=d1, out_ld=32, relu_mask=act1[0], colsum=cs1)
    got1 = d1.float().sum(0).view(B, hp1, 21, 32)
    np.testing.assert_allclose(got1[:, off1:off1 + 21].cpu().numpy(), want1.cpu().numpy(), rtol=0, atol=atol * 4)
    assert float(got1[:, :off1].abs().max()) == 0.0 and off1 + 21 == hp1
    np.testing.assert_allclose(tc.bias_grad(cs1, 32).cpu().numpy(), want1.sum((0, 1, 2)).cpu().numpy(), rtol=0, atol=atol * 8000)


@pytest.mark.parametrize("planes,fwd_tol,grad_tol", [(2, 1e-4, 2e-2), (3, 2e-5, 2e-3)])
def test_encoder_matches_cudnn_fp32(planes, fwd_tol, grad_tol):
    """Whole encoder forward + backward vs the cuDNN fp32 path.  Per-layer gradients with a given mask are pinned above; here
    the masks come from each network's own activations, so a pre-activation within ~1e-5 (two planes) / ~1e-6 (three) of
    zero can take the other side of its ReLU than in the cuDNN network and move the upstream gradients by O(1/B) - the
    comparison is therefore in norm."""
    from helpers import build_product_ppo_model
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(1)
    m_ref = build_product_ppo_model(4, DEV).to(DEV)
    m_tc = build_product_ppo_model(4, DEV).to(DEV)
    m_tc.load_state_dict(m_ref.state_dict())
    m_tc.representation.tc_planes = planes
    m_tc.representation.set_compute("tc")
    obs = torch.randint(0, 256, (64, 84, 84, 4), dtype=torch.uint8, device=DEV)
    R = torch.randn(64, 512, device=DEV)
    z_ref = m_ref.representation(obs).embeddings
    z_tc = m_tc.representation(obs).embeddings
    np.testing.assert_allclose(z_tc.detach().cpu().numpy(), z_ref.detach().cpu().numpy(), rtol=fwd_tol, atol=fwd_tol)
    (z_ref * R).sum().backward()
    (z_tc * R).sum().backward()
    for (k, p), (_, q) in zip(m_ref.representation.named_parameters(), m_tc.representation.named_parameters()):
        rel = float((q.grad - p.grad).norm() / p.grad.norm())
        assert rel < grad_tol, (k, rel)


@pytest.mark.parametrize("planes", [1, 2, 3])
def test_gather_obs_planes(planes):
    """K3-P: uint8 rows gathered straight into bf16 planes - of x/255 (true float32 division, as the reference's
    `observations / 255.0` on the host) for 2 / 3 planes, of the raw pixel value for 1 plane; bit-exact."""
    from xuance_b200 import _lib
    buf = torch.randint(0, 256, (6, 5, 84, 84, 4), dtype=torch.uint8, device=DEV)
    idx = torch.tensor([29, 0, 7, 7, 13, 1, 28], dtype=torch.int64, device=DEV)
    out = torch.empty((planes, idx.numel(), 84, 84, 4), dtype=torch.bfloat16, device=DEV)
    _lib.call("xb_gather_obs_planes", _lib.ptr(buf), _lib.ptr(idx), idx.numel(), 84 * 84 * 4, planes, _lib.ptr(out))
    rows = buf.reshape(-1, 84, 84, 4)[idx].cpu().float()
    val = rows if planes == 1 else torch.from_numpy(rows.numpy() / np.float32(255.0))   # IEEE division on the host
    assert torch.equal(out.cpu(), _planes_ref(val, planes))
    out2 = torch.empty((planes, 30, 84, 84, 4), dtype=torch.bfloat16, device=DEV)
    _lib.call("xb_gather_obs_planes", _lib.ptr(buf), None, 30, 84 * 84 * 4, planes, _lib.ptr(out2))
    allv = buf.reshape(-1, 84, 84, 4).cpu().float()
    allv = allv if planes == 1 else torch.from_numpy(allv.numpy() / np.float32(255.0))
    assert torch.equal(out2.cpu(), _planes_ref(allv, planes))


def test_ppo_update_tc_three_planes_matches_fp32():
    """PPO_Learner.update with compute='tc' (three planes) next to the cuDNN fp32 learner: same losses, same parameters."""
    from helpers import build_product_ppo_model, ppo_config
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import PPO_Learner
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(3)
    A, B = 6, 256
    m_ref = build_product_ppo_model(A, DEV)
    m_tc = build_product_ppo_model(A, DEV)
    m_tc.load_state_dict(m_ref.state_dict())
    m_tc.representation.tc_planes = 3
    m_tc.representation.set_compute("tc")
    cfg = ppo_config(DEV, running_steps=256 * 128 * 10)
    l_ref, l_tc = PPO_Learner(cfg, m_ref, BaseCallback()), PPO_Learner(cfg, m_tc, BaseCallback())
    rng = np.random.default_rng(5)
    for it in range(3):
        s = {"obs": torch.from_numpy(rng.integers(0, 256, size=(B, 84, 84, 4), dtype=np.uint8)).cuda(),
             "actions": rng.integers(0, A, size=B).astype(np.float32), "returns": rng.normal(size=B).astype(np.float32),
             "advantages": rng.normal(size=B).astype(np.float32),
             "aux_batch": {"old_logp": (rng.normal(size=B) * 0.05 - np.log(A)).astype(np.float32)}}
        i_ref, i_tc = l_ref.update(**s), l_tc.update(**s)
        for k in ("actor_loss", "critic_loss", "entropy", "predict_value"):
            np.testing.assert_allclose(i_tc[k], i_ref[k], rtol=2e-4, atol=1e-5, err_msg=k)
    for (k, p), (_, q) in zip(m_ref.state_dict().items(), m_tc.state_dict().items()):
        np.testing.assert_allclose(q.cpu().numpy(), p.cpu().numpy(), rtol=1e-3, atol=1e-4, err_msg=k)

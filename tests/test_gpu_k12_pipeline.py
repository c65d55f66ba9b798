"""Edges of the K12 persistent consumer loop (xuance_b200/csrc/conv_tc.cu) where its control flow turns, against float64
references with the tolerances of test_gpu_tc_conv.py: one, two and an odd number of 64-deep chunks per item, fewer work
items than CTAs, one more item than CTAs and an odd number per CTA, halo launches with one and four sub-items, a
weight-gradient split whose last run is a single chunk, the fused ReLU mask and column sums - and two launches of the same
inputs must agree bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PLANES, ATOL = 3, 3e-6


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _linear(B, K, N, seed, mask=False):
    """Linear forward (TMA tiles) with bias + ReLU, optionally with a ReLU-derivative mask and the column sums; returns a
    function that launches it (-> float32 result, column sums or None) and the float64 reference."""
    from xuance_b200.torch.utils import tc_conv as tc
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.rand(B, K, device=DEV, generator=g)
    w = torch.randn(N, K, device=DEV, generator=g) / np.sqrt(K)
    b = torch.randn(N, device=DEV, generator=g) * 0.1
    want = F.relu(x.double() @ w.double().t() + b.double())
    kw = {}
    if mask:
        m = tc.split_bf16(torch.randn(B, N, device=DEV, generator=g), PLANES)[0]
        kw = dict(relu_mask=m, mask_ld=N, mask_c0=0, colsum=torch.full((-(-B // 128), N), float("nan"), device=DEV))
        want = want * (m.float() > 0)

    def run():
        out = torch.full((B, N), float("nan"), device=DEV)
        cs = kw.get("colsum")
        if cs is not None:
            kw["colsum"] = torch.full_like(cs, float("nan"))
        tc.gemm_gather(tc.split_bf16(x, PLANES), tc.split_bf16(w, PLANES), tc.linear_geometry(B, K), bias=b, relu=True,
                       out_f32=out, **kw)
        return out, kw.get("colsum")
    return run, want


@pytest.mark.parametrize("N", [32, 64])
@pytest.mark.parametrize("K", [64, 128, 576])
def test_chunks_per_item(K, N):
    """1, 2 and 9 chunks per work item, 32- and 64-column tiles."""
    run, want = _linear(300, K, N, seed=K + N)
    out, _ = run()
    np.testing.assert_allclose(out.cpu().numpy(), want.cpu().numpy(), rtol=0, atol=ATOL)


@pytest.mark.parametrize("items", ["fewer_than_ctas", "ctas_plus_one", "odd_per_cta"])
def test_work_items_per_cta(items):
    sm = _sm_count()
    tiles = {"fewer_than_ctas": 2, "ctas_plus_one": sm + 1, "odd_per_cta": 2 * sm + 1}[items]
    B = 128 * tiles - 5                                       # the last M tile is partial
    run, want = _linear(B, 192, 32, seed=tiles)
    out, _ = run()
    np.testing.assert_allclose(out.cpu().numpy(), want.cpu().numpy(), rtol=0, atol=ATOL)


@pytest.mark.parametrize("N", [32, 64])
def test_mask_and_column_sums_bit_identical_across_launches(N):
    run, want = _linear(128 * 5 + 17, 576, N, seed=7, mask=True)
    out, cs = run()
    np.testing.assert_allclose(out.cpu().numpy(), want.cpu().numpy(), rtol=0, atol=ATOL)
    tiles = want.new_zeros(cs.shape[0] * 128, N)
    tiles[:want.shape[0]] = want
    np.testing.assert_allclose(cs.cpu().numpy(), tiles.view(-1, 128, N).sum(1).cpu().numpy(), rtol=0, atol=ATOL * 200)
    out2, cs2 = run()
    assert torch.equal(out, out2) and torch.equal(cs, cs2)


def test_weight_gradient_last_split_one_chunk():
    """400 sites in 3 splits of 192: the last run holds 16 sites, one chunk; the others three chunks each."""
    from xuance_b200.torch.utils import tc_conv as tc
    g = torch.Generator(device=DEV).manual_seed(3)
    M, K, N, splits = 400, 256, 64, 3
    x = torch.rand(M, K, device=DEV, generator=g)
    gy = torch.randn(M, N, device=DEV, generator=g) / 16
    want = (gy.double().t() @ x.double()).cpu().numpy()
    geom = tc.linear_geometry(M, K)
    dws = []
    for _ in range(2):
        part = tc.wgrad_gather(tc.split_bf16(x, PLANES), tc.split_bf16(gy, PLANES), geom, splits)
        dws.append(tc.wgrad_reduce(part, N, K, 1, 1).reshape(N, K))
    np.testing.assert_allclose(dws[0].cpu().numpy(), want, rtol=0, atol=2e-5)
    assert torch.equal(dws[0], dws[1])


@pytest.mark.parametrize("B", [1, 7])
def test_halo_one_and_four_sub_items(B):
    """conv3 forward (one sub-item, 9 chunks) and conv2's data gradient (four stride phases as sub-items of one resident
    tile, 4 chunks each) with mask and column sums; B = 1 gives fewer M tiles than CTAs."""
    import torch.nn as nn
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(17)
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    enc = tc.BoxNatureCNN([c.to(DEV) for c in convs], None, (84, 84, 4), backend=tc.CudaBackend(PLANES))
    P = enc._plan(B)
    hp1, hp2, off1, W1p, xo1 = P["hp1"], P["hp2"], P["off1"], P["W1p"], P["xo1"]
    w2, w3, b3 = convs[1].weight.detach(), convs[2].weight.detach(), convs[2].bias.detach()
    pad2 = lambda t: torch.cat([torch.zeros_like(t[:, :, :1]), t, torch.zeros_like(t[:, :, :1])], 2).reshape(PLANES, B * hp2, 10, 64)
    a2 = torch.rand(B, 10, 10, 64, device=DEV)
    act2 = pad2(tc.split_bf16(a2, PLANES))
    w3p = tc.pack_conv_weight(w3, PLANES)
    outs = []
    for _ in range(2):
        out3 = torch.full((B * 100, 64), float("nan"), device=DEV)
        tc.gemm_halo(act2, w3p, P["h_fwd3"], bias=b3, relu=True, out_f32=out3, out_ld=64)
        outs.append(out3)
    want3 = F.relu(F.conv2d(a2.permute(0, 3, 1, 2).double(), w3.double(), b3.double(), stride=1, padding=1)).permute(0, 2, 3, 1)
    np.testing.assert_allclose(outs[0].view(B, 10, 10, 64).cpu().numpy(), want3.cpu().numpy(), rtol=0, atol=ATOL)
    assert torch.equal(outs[0], outs[1])
    a1 = torch.rand(B, 21, 21, 32, device=DEV) - 0.3
    act1 = torch.zeros(PLANES, B, hp1, W1p, 32, dtype=torch.bfloat16, device=DEV)
    act1[:, :, off1:off1 + 21, xo1:xo1 + 21] = tc.split_bf16(a1, PLANES)
    act1 = act1.view(PLANES, B * hp1, W1p, 32)
    g2 = torch.randn(B, 10, 10, 64, device=DEV)
    g2p = pad2(tc.split_bf16(g2, PLANES))
    x1 = a1.double().permute(0, 3, 1, 2).requires_grad_(True)
    (dx1,) = torch.autograd.grad(F.conv2d(x1, w2.double(), stride=2, padding=1), x1, g2.double().permute(0, 3, 1, 2))
    want1 = dx1.permute(0, 2, 3, 1) * (act1[0].float().view(B, hp1, W1p, 32)[:, off1:off1 + 21, xo1:xo1 + 21] > 0)
    wd2 = torch.cat([tc.split_bf16(tc.dgrad_weight_matrix(w2, taps), PLANES) for _, taps in P["dg2"]], 1).contiguous()
    res = []
    for _ in range(2):
        d1 = torch.zeros(PLANES, B * hp1, 21, 32, dtype=torch.bfloat16, device=DEV)
        cs1 = torch.full((P["h_dg2"].m_tiles, 32), float("nan"), device=DEV)
        tc.gemm_halo(g2p, wd2, P["h_dg2"], out_pl=d1, out_ld=32, relu_mask=act1[0], colsum=cs1)
        res.append((d1, cs1))
    got1 = res[0][0].float().sum(0).view(B, hp1, 21, 32)
    np.testing.assert_allclose(got1[:, off1:off1 + 21].cpu().numpy(), want1.cpu().numpy(), rtol=0, atol=ATOL * 4)
    np.testing.assert_allclose(tc.bias_grad(res[0][1].clone(), 32).cpu().numpy(), want1.sum((0, 1, 2)).cpu().numpy(), rtol=0,
                               atol=ATOL * 8000)
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])

"""CPU: the exact references of tests/k12_exact_refs.py - the float64 weight-gradient references against
``torch.nn.grad.conv2d_weight`` at every production geometry, the operand builders' premise, the float32 restatement of
xb_wgrad_reduce against a float64 sum, and the launch recorder and replay on the CPU-restated launches of
tests/test_k12_geometry.py."""
import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_weight

import k12_exact_refs as X
from test_k12_geometry import _encoder_modules, _planes_ref, host_k12  # noqa: F401  (host_k12 is a fixture)
from xuance_b200.torch.utils import tc_conv as tc


def _plan(B):
    convs, fc = _encoder_modules()
    return tc.BoxNatureCNN(convs, fc, (84, 84, 4), backend=tc.CudaBackend(3))._plan(B)


def _pl(t):
    return t.to(torch.bfloat16)[None]


def _check_splits(ref, full_fn, g, per, splits):
    """Split s of ``ref`` equals the one-split reference of g restricted to the sites of split s."""
    flat = g.reshape(g.shape[0], -1, g.shape[-1])
    for s in sorted({0, splits // 2, splits - 1}):
        m = torch.zeros_like(flat)
        m[:, s * per:(s + 1) * per] = flat[:, s * per:(s + 1) * per]
        torch.testing.assert_close(ref[s], full_fn(m.view(g.shape))[0], rtol=1e-12, atol=1e-12)


def test_references_equal_conv2d_weight_at_every_production_geometry():
    B = 2
    P = _plan(B)
    gen = torch.Generator().manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64).bfloat16().double()
    nchw = lambda t: t.permute(0, 3, 1, 2)
    hp1, hp2, off1, xo1, W1p = P["hp1"], P["hp2"], P["off1"], P["xo1"], P["W1p"]
    # conv1 over the raw input, its gradient on act1's padded grid (the padding rows zero)
    x0, g1 = r(B, 84, 84, 4), r(B, 21, 21, 32)
    gp = torch.zeros(B, hp1, 21, 32, dtype=torch.float64)
    gp[:, off1:off1 + 21] = g1
    geom = P["wg1"]
    splits = tc.wgrad_splits(geom.M, geom.K)
    ref = X.wgrad_gather_ref(_pl(x0), _pl(gp.reshape(geom.M, 32)), geom, splits)
    want = conv2d_weight(nchw(x0), (32, 4, 8, 8), nchw(g1), stride=4, padding=2)
    torch.testing.assert_close(X.torch_layout(ref.sum(0), 32, 4, 8, 8), want, rtol=1e-12, atol=1e-10)
    _check_splits(ref, lambda g: X.wgrad_gather_ref(_pl(x0), g, geom, 1), _pl(gp.reshape(geom.M, 32)), X.sites_per_split(geom.M, splits), splits)
    # conv2 gathered and box (pixel pairs): act1 padded, its padding NON-zero (it must not reach the result through a zero g)
    a1, g2 = r(B, 21, 21, 32), r(B, 10, 10, 64)
    xa = r(B, hp1, W1p, 32)
    xa[:, off1:off1 + 21, xo1:xo1 + 21] = a1
    x_real = torch.zeros_like(xa)
    x_real[:, off1:off1 + 21, xo1:xo1 + 21] = a1
    gq = torch.zeros(B, hp2, 10, 64, dtype=torch.float64)
    gq[:, 1:11] = g2
    want = conv2d_weight(nchw(a1), (64, 32, 4, 4), nchw(g2), stride=2, padding=1)
    ref = X.wgrad_gather_ref(_pl(x_real), _pl(gq.reshape(-1, 64)), P["wg2"], 2)
    torch.testing.assert_close(X.torch_layout(ref.sum(0), 64, 32, 4, 4), want, rtol=1e-12, atol=1e-10)
    ref = X.wgrad_box_ref(_pl(x_real.reshape(B * hp1, W1p // 2, 64)), _pl(gq.reshape(B * hp2, 10, 64)), P["fwd2"], 6, 2)
    torch.testing.assert_close(X.torch_layout(ref.sum(0), 64, 32, 4, 4), want, rtol=1e-12, atol=1e-10)
    # the padding of the input changes the result only where g is non-zero on a padding site: zero here
    ref_pad = X.wgrad_box_ref(_pl(xa.reshape(B * hp1, W1p // 2, 64)), _pl(gq.reshape(B * hp2, 10, 64)), P["fwd2"], 6, 2)
    assert not torch.equal(ref_pad, ref), "the box reference does not read act1's padding"
    # conv3 gathered and box
    a2, g3 = r(B, 10, 10, 64), r(B, 10, 10, 64)
    xb = torch.zeros(B, hp2, 10, 64, dtype=torch.float64)
    xb[:, 1:11] = a2
    gb = torch.zeros(B, hp2, 10, 64, dtype=torch.float64)
    gb[:, 1:11] = g3
    want = conv2d_weight(nchw(a2), (64, 64, 3, 3), nchw(g3), stride=1, padding=1)
    for ref in (X.wgrad_gather_ref(_pl(xb), _pl(gb.reshape(-1, 64)), P["wg3"], 2),
                X.wgrad_box_ref(_pl(xb.reshape(-1, 10, 64)), _pl(gb.reshape(-1, 10, 64)), P["fwd3"], 6, 4)):
        torch.testing.assert_close(X.torch_layout(ref.sum(0), 64, 64, 3, 3), want, rtol=1e-12, atol=1e-10)
    # the Linear layer: [(h, w, c)] input rows, torch's [N, (c, h, w)] weight
    a3, gy = r(B, 10, 10, 64), r(B, 512)
    ref = X.wgrad_gather_ref(_pl(a3.reshape(B, 6400)), _pl(gy), P["fc"]["fwd"], 1)
    want = gy.t() @ nchw(a3).reshape(B, 6400)
    torch.testing.assert_close(X.torch_layout(ref.sum(0), 512, 64, 10, 10).reshape(512, 6400), want, rtol=1e-12, atol=1e-10)


def test_kept_products_are_those_with_plane_index_sum_below_pb():
    gen = torch.Generator().manual_seed(1)
    geom = tc.linear_geometry(64, 64)
    x = X.fill((64, 64), 3, "sparse", gen, 0.5, signed=False, device="cpu")
    g = X.fill((64, 32), 3, "sparse", gen, 0.5, device="cpu")
    want = sum(x[i].double().t() @ g[j].double() for i in range(3) for j in range(3) if i + j < 3)
    torch.testing.assert_close(X.wgrad_gather_ref(x, g, geom, 1)[0], want, rtol=0, atol=0)
    x1 = x[:1]                                          # one raw plane meets all three planes of g
    torch.testing.assert_close(X.wgrad_gather_ref(x1, g, geom, 1)[0], x1[0].double().t() @ g.double().sum(0), rtol=0, atol=0)


@pytest.mark.parametrize("mode", ["dense", "sparse"])
def test_builders_satisfy_the_premise(mode):
    """At B = 2 the premise is computed; at B = 8192 (the largest production batch) every weight gradient keeps the dense
    fill at full density and the expected sum is one bit below the limit (the GPU test computes the premise itself)."""
    B = 2
    P = _plan(B)
    gen = torch.Generator().manual_seed(2)
    for key, N in (("wg1", 32), ("wg2", 64), ("wg3", 64)):
        geom = P[key]
        pa = 1 if key == "wg1" else 3
        x = X.fill((geom.B, geom.IH, geom.IW, geom.C), pa, mode, gen, 0.5, signed=False, device="cpu")
        g = X.fill((geom.M, N), 3, mode, gen, X.density_for(geom.M, mode), device="cpu")
        mag = X.wgrad_gather_ref(x.abs(), g.abs(), geom, 1)
        X.check_premise(mag.sum(0), 1.0 if mode == "dense" else 2.0 ** -4, key)
    Pl = _plan(8192)
    for geom in (Pl["wg1"], Pl["wg2"], Pl["wg3"], Pl["fc"]["fwd"]):
        if mode == "dense":
            assert X.density_for(geom.M, mode) == 1.0 and geom.M <= X.LIMIT     # every |term| <= 1: sum <= M
        d = X.density_for(geom.M, mode)
        assert geom.M * 0.5 * d * (16.0 / 9.0 if mode == "sparse" else 1.0) <= X.LIMIT / 2 * (1.0 if mode == "dense" else 2.0 ** -4) * 1.0001


def test_premise_check_rejects_a_breaking_operand():
    X.check_premise(torch.tensor([2.0 ** 22]), 1.0, "at the limit")
    with pytest.raises(AssertionError, match="exactness premise broken"):
        X.check_premise(torch.tensor([2.0 ** 22 + 1]), 1.0, "one above")
    geom = tc.linear_geometry(2 ** 12 + 64, 64)
    x = torch.ones((1, geom.M, 64), dtype=torch.bfloat16)
    g = torch.full((1, geom.M, 32), 2.0 ** 10, dtype=torch.bfloat16)                 # 4160 * 1024 > 2^22
    with pytest.raises(AssertionError, match="exactness premise broken"):
        X.check_premise(X.wgrad_gather_ref(x, g, geom, 1).sum(0), 1.0, "dense ones")


@pytest.mark.parametrize("splits,N,C,KH,KW,kind", [
    (1009, 32, 4, 8, 8, "fold+lane"), (257, 64, 32, 4, 4, "fold+lane"), (36864, 32, 1, 1, 1, "fold+lane"),
    (2, 512, 64, 10, 10, "tiled"), (16, 512, 64, 10, 10, "tiled"), (17, 512, 64, 10, 10, "lane"),
    (30, 64, 64, 3, 3, "lane"), (1, 64, 32, 4, 4, "lane"), (256, 32, 1, 1, 1, "lane")])
def test_reduce_restatement_is_exact_on_exact_partials(splits, N, C, KH, KW, kind):
    gen = torch.Generator().manual_seed(splits)
    K = C * KH * KW
    p = torch.randint(-64, 65, (splits, K, N), generator=gen).float()
    assert X.reduce_kind(splits, N, C, KH, KW) == kind
    want = X.torch_layout(p.double().sum(0).float(), N, C, KH, KW)
    torch.testing.assert_close(X.reduce_ref(p, N, C, KH, KW, sm_count=132), want, rtol=0, atol=0)
    prev = torch.randn(N, C, KH, KW, generator=gen)
    torch.testing.assert_close(X.reduce_ref(p, N, C, KH, KW, out=prev, accumulate=True, sm_count=132), prev + want, rtol=0, atol=0)
    s = X.reduce_ref(p, N, C, KH, KW, scale=1.0 / 255.0, sm_count=132)
    torch.testing.assert_close(s, X.reduced_ref(p.double(), N, C, KH, KW, 1.0 / 255.0), rtol=0, atol=0)


def test_reduce_restatement_follows_the_kernel_order():
    """On arbitrary float32 partials the order matters: the lane kernel's strided sums differ from a sequential sum."""
    gen = torch.Generator().manual_seed(3)
    p = torch.randn(64, 64, 64, generator=gen) * torch.logspace(-6, 6, 64)[:, None, None]
    lanes = X.lanes_for(64, 1, 64 * 64, 132)
    assert lanes > 1
    seq = torch.zeros(64 * 64)
    for k in range(64):
        seq = seq + p[k].reshape(-1)
    got = X.reduce_ref(p, 64, 64, 1, 1, sm_count=132).permute(2, 3, 1, 0).reshape(-1)
    assert not torch.equal(got, seq)
    strided = [torch.zeros(64 * 64) for _ in range(lanes)]
    for k in range(64):
        strided[k % lanes] = strided[k % lanes] + p[k].reshape(-1)
    want = strided[0]
    for q in range(1, lanes):
        want = want + strided[q]
    assert torch.equal(got, want)


def _run(enc, B, gen):
    x_pl = _planes_ref(torch.randint(0, 256, (B, 84, 84, 4), generator=gen).float(), 1)
    z = tc.tc_encode(enc, x_pl, B)
    z.backward(torch.randn(z.shape, generator=gen))


RESTATED = lambda: {n: getattr(tc, n) for n in X.Recorder.NAMES}
BIAS_GRAD = tc.bias_grad          # the product's: it reaches wgrad_reduce through the module, where the recorder sits


@pytest.mark.parametrize("halo,box_wgrad", [("2", "3"), ("0", ""), ("3", "23")])
def test_recorder_and_replay_on_restated_launches(host_k12, halo, box_wgrad):
    """The recorder on BoxNatureCNN.backward over the restated launches: one chain per weight and per K12 bias gradient,
    the split counts of the split rules, conv1's 1/255, the padding rows of conv1's output gradient outside the support;
    then the replay through the same restated launches runs clean in the dense filling."""
    host_k12.setattr(tc, "HALO", halo != "0")
    host_k12.setattr(tc, "HALO3", halo == "3")
    host_k12.setattr(tc, "BOX_WGRAD2", "2" in box_wgrad)
    host_k12.setattr(tc, "BOX_WGRAD3", "3" in box_wgrad)
    host_k12.setattr(tc, "bias_grad", BIAS_GRAD)
    B = 2
    convs, fc = _encoder_modules()
    enc = tc.BoxNatureCNN(convs, fc, (84, 84, 4), backend=tc.CudaBackend(3))
    launches = RESTATED()
    rec = X.Recorder(host_k12)
    _run(enc, B, torch.Generator().manual_seed(4))
    chains = rec.chains()
    wg = [(p[0], r) for p, r in chains if p[0]["kind"].startswith("wgrad")]
    cs = [(p, r) for p, r in chains if p[0]["kind"].startswith("gemm")]
    assert [r["N"] * r["C"] * r["KH"] * r["KW"] for _, r in wg] == [512 * 6400, 64 * 576, 64 * 512, 32 * 256]
    assert [p["kind"] for p, _ in wg] == ["wgrad_gather", "wgrad_box" if "3" in box_wgrad else "wgrad_gather",
                                         "wgrad_box" if "2" in box_wgrad else "wgrad_gather", "wgrad_gather"]
    assert [r["scale"] for _, r in wg] == [1.0, 1.0, 1.0, pytest.approx(1.0 / 255.0)]
    assert [len(p) for p, _ in cs] == [1, 1, 1 if halo != "0" else 4]
    assert [r["N"] for _, r in cs] == [64, 64, 32] and all(r["C"] == r["KH"] == r["KW"] == 1 for _, r in cs)
    P = enc._plan(B)
    for p, r in wg:
        if p["kind"] == "wgrad_gather":
            assert p["splits"] == tc.wgrad_splits(p["geom"].M, p["geom"].K, r["N"] // tc.n_tile_for(r["N"], 3))
        else:
            assert p["splits"] == tc.wgrad_box_splits(B * P["hp2"], 6, p["geom"].K, r["N"])
    sup1 = wg[3][0]["support"].view(B, P["hp1"], P["W1"])
    assert not sup1[:, :P["off1"]].any() and not sup1[:, P["off1"] + P["H1"]:].any() and sup1[:, P["off1"]:P["off1"] + P["H1"]].all()
    worst = X.replay(rec, launches, modes=("dense",), sm_count=132)
    assert len(worst) == len(chains) and all(0 < v <= X.LIMIT for v in worst.values())
    # the restated weight gradients multiply every pair of planes; the launches drop plane-index sums >= PB, and the
    # sparse fill sees the difference
    with pytest.raises(AssertionError, match="sparse.*partials"):
        X.replay(rec, launches, modes=("sparse",), sm_count=132)


def test_recorder_on_the_gathered_encoder(host_k12):
    convs, fc = _encoder_modules(seed=1)
    enc = tc.TensorCoreNatureCNN(convs, fc, (84, 84, 4), backend=tc.CudaBackend(3))
    launches = RESTATED()
    rec = X.Recorder(host_k12)
    _run(enc, 2, torch.Generator().manual_seed(5))
    chains = rec.chains()
    assert [p[0]["kind"] for p, _ in chains] == ["wgrad_gather"] * 4
    X.replay(rec, launches, modes=("dense",), sm_count=132)

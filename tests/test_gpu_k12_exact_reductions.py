"""GPU: K12's weight- and bias-gradient reductions bit for bit on exactly representable operands (tests/k12_exact_refs.py
derives why the kernels must then return the float64 value exactly, whatever order they sum in).

  * Production replay: one ordinary backward of the encoder with every reduction launch recorded (split partials, column
    sums, reduces), then every recorded launch again with exact operands of the same shapes, strides, geometries, split
    counts and scales - at the agents' batch sizes, Basic_CNN, two planes, every XB_K12_HALO x XB_K12_BOX_WGRAD path,
    TensorCoreNatureCNN and XB_K12_TMA=0.  A change of a plan or a split rule is followed without edits.
  * Launch level: split counts beyond what production picks (1, the rule's, a one-chunk tail, counts above 256 with a
    partial last fold group, the largest the rule allows) for every weight-gradient path, and xb_wgrad_reduce on random
    float32 partials against its order-exact restatement.
  * A premise probe first: a sum that needs all 24 bits of a float32."""
import json
import os
import subprocess
import sys

import pytest
import torch

import k12_exact_refs as X
from test_k12_geometry import _encoder_modules
from xuance_b200.torch.utils import tc_conv as tc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_premise_probe_a_sum_needing_all_24_bits():
    """Every column sums the 23 powers 2^0 .. 2^22 (= 2^23 - 1) over 64 sites, in a different site order per column: exact
    only if the tensor core's truncating add keeps every bit of a sum below 2^24 (DESIGN.md section 4)."""
    gen = torch.Generator().manual_seed(0)
    geom = tc.linear_geometry(64, 64)
    g = torch.zeros(64, 32)
    for n in range(32):
        order = torch.arange(23) if n == 0 else torch.arange(22, -1, -1) if n == 1 else torch.randperm(23, generator=gen)
        sites = torch.randperm(64, generator=gen)[:23] if n > 1 else torch.arange(23)
        g[sites, n] = torch.pow(2.0, order.float())
    x = torch.ones((1, 64, 64), dtype=torch.bfloat16, device=DEV)
    part = tc.wgrad_gather(x, g.to(DEV).bfloat16()[None], geom, 1)
    bad = int((part != 2.0 ** 23 - 1).sum())
    assert bad == 0, ("premise broken: %d of %d sums of 2^0 .. 2^22 are not 2^23 - 1 (largest error %g): the tensor core does "
                      "not add representable values exactly below 2^24, so the exact comparisons of this file do not hold "
                      "as derived" % (bad, part.numel(), float((part.double() - (2.0 ** 23 - 1)).abs().max())))


# ------------------------------------------------------------------------------------------------ production replay
def _encoder(basic=False, cls=tc.BoxNatureCNN, planes=3, seed=0):
    convs, fc = _encoder_modules(0 if basic else 512, seed)
    return cls([c.to(DEV) for c in convs], fc.to(DEV) if fc is not None else None, (84, 84, 4), backend=tc.CudaBackend(planes))


def _expected(enc):
    """Producer kinds of each reduce of one backward, in order."""
    if type(enc) is tc.TensorCoreNatureCNN:
        return ["wgrad_gather"] * (4 if enc.fc is not None else 3)
    box3, box2 = ("wgrad_box" if f else "wgrad_gather" for f in (tc.BOX_WGRAD3, tc.BOX_WGRAD2))
    dg3 = "gemm_halo" if tc.HALO3 else "gemm_box"
    dg2 = "gemm_halo" if tc.HALO else "gemm_box"
    head = ["wgrad_gather", "gemm_gather"] if enc.fc is not None else []
    return head + [box3, dg3, box2, dg2, "wgrad_gather"]


def _record_and_replay(monkeypatch, enc, B, seed=0):
    rec = X.Recorder(monkeypatch)
    gen = torch.Generator(device=DEV).manual_seed(seed + B)
    obs = torch.randint(0, 256, (B, 84, 84, 4), device=DEV, generator=gen)
    x_pl = obs.to(torch.bfloat16)[None]                                   # the raw uint8 pixels as one exact plane
    z = tc.tc_encode(enc, x_pl, B)
    z.backward(torch.randn(z.shape, device=DEV, generator=gen))
    torch.cuda.synchronize()
    chains = rec.chains()
    assert ["+".join(sorted({p["kind"] for p in prods})) for prods, _ in chains] == _expected(enc), \
        "a layer's reduction was not launched as the plan says: %s" % [[p["kind"] for p in prods] for prods, _ in chains]
    worst = X.replay(rec, rec.orig, seed=seed + B, sm_count=_sm())
    print("B=%d (reduce order for %d SMs) largest sum|terms|/res (limit 2^22 = %d): %s"
          % (B, _sm(), int(X.LIMIT), json.dumps({"%s %s" % k: int(v) for k, v in worst.items()})))
    return worst


@pytest.mark.parametrize("B", [1, 2, 37, 255, 256, 257, 1024, 2731, 8192])
def test_production_launches_exact(monkeypatch, B):
    _record_and_replay(monkeypatch, _encoder(), B)


@pytest.mark.parametrize("B", [32, 512])
def test_basic_cnn_launches_exact(monkeypatch, B):
    _record_and_replay(monkeypatch, _encoder(basic=True), B)


@pytest.mark.parametrize("B", [37, 2731])
def test_two_plane_launches_exact(monkeypatch, B):
    _record_and_replay(monkeypatch, _encoder(planes=2), B)


@pytest.mark.parametrize("B", [37, 2731])
@pytest.mark.parametrize("box_wgrad", ["", "2", "3", "23"])
@pytest.mark.parametrize("halo", ["0", "2", "3"])
def test_path_switch_launches_exact(monkeypatch, halo, box_wgrad, B):
    monkeypatch.setattr(tc, "HALO", halo != "0")
    monkeypatch.setattr(tc, "HALO3", halo == "3")
    monkeypatch.setattr(tc, "BOX_WGRAD2", "2" in box_wgrad)
    monkeypatch.setattr(tc, "BOX_WGRAD3", "3" in box_wgrad)
    _record_and_replay(monkeypatch, _encoder(), B)


@pytest.mark.parametrize("basic", [False, True])
@pytest.mark.parametrize("B", [37, 2731])
def test_gathered_encoder_launches_exact(monkeypatch, B, basic):
    """TensorCoreNatureCNN: CudaBackend.wgrad (its bias gradients are torch column sums, not K12 launches)."""
    _record_and_replay(monkeypatch, _encoder(basic=basic, cls=tc.TensorCoreNatureCNN), B)


# ------------------------------------------------------------------------------------------------ launch level
def _desc(shape):
    t = torch.empty(shape, dtype=torch.bfloat16, device="meta")
    return dict(shape=tuple(shape), stride=t.stride(), dtype=torch.bfloat16)


def _launch(path, B):
    """(producer, reduce, sites or rows, unit) of one weight-gradient launch of BoxNatureCNN's plan, as the recorder keeps
    them; the support marks the real rows of the padded output-gradient grid."""
    convs, fc = _encoder_modules()
    P = tc.BoxNatureCNN(convs, fc, (84, 84, 4), backend=tc.CudaBackend(3))._plan(B)
    ones = lambda *s: torch.ones(s, dtype=torch.bool, device=DEV)
    real = ones(B, P["hp2"], P["W2"])
    real[:, 0] = real[:, 1 + P["H2"]:] = False
    if path == "wg1":
        geom = P["wg1"]
        sup = ones(B, P["hp1"], P["W1"])
        sup[:, :P["off1"]] = sup[:, P["off1"] + P["H1"]:] = False
        prod = dict(kind="wgrad_gather", geom=geom, n_tile=None, x=_desc((1, B * 84 * 84 * 4)), g=_desc((3, geom.M, 32)), support=sup.view(-1))
        red = dict(N=32, C=4, KH=8, KW=8, scale=1.0 / 255.0)
    elif path in ("wg2", "wg3"):
        geom = P[path]
        prod = dict(kind="wgrad_gather", geom=geom, n_tile=None, x=_desc((3, geom.B * geom.IH, geom.IW, geom.C)), g=_desc((3, geom.M, 64)),
                    support=real.view(-1))
        red = dict(N=64, C=geom.C, KH=4 if path == "wg2" else 3, KW=4 if path == "wg2" else 3, scale=1.0)
    elif path == "fc":
        geom = P["fc"]["fwd"]
        prod = dict(kind="wgrad_gather", geom=geom, n_tile=None, x=_desc((3, B, 6400)), g=_desc((3, B, 512)), support=ones(B))
        red = dict(N=512, C=64, KH=10, KW=10, scale=1.0)
    else:
        bg = P["fwd2" if path == "box2" else "fwd3"]
        prod = dict(kind="wgrad_box", geom=bg, box_h=6, x=_desc((3, bg.B * bg.hp_in, bg.W, bg.C)), g=_desc((3, B * P["hp2"], P["W2"], 64)),
                    support=real.view(B * P["hp2"], P["W2"]))
        red = dict(N=64, C=32 if path == "box2" else 64, KH=4 if path == "box2" else 3, KW=4 if path == "box2" else 3, scale=1.0)
        return prod, red, B * P["hp2"], 6
    return prod, red, geom.M, tc.KC


def _split_counts(path, prod, red, units, unit):
    if prod["kind"] == "wgrad_box":
        rule = tc.wgrad_box_splits(units, unit, prod["geom"].K, red["N"])
    else:
        rule = tc.wgrad_splits(units, prod["geom"].K, red["N"] // tc.n_tile_for(red["N"], 3))
    top = X.max_splits(units, unit)
    valid = (lambda s: X.box_rows_per_split(units, s, unit) > 0) if prod["kind"] == "wgrad_box" else (lambda s: X.sites_per_split(units, s) > 0)
    counts = {1, rule, top} | {s for s in (257, 1009) if s <= top and valid(s)}
    if units > unit:
        counts.add(X.single_chunk_tail(units, unit))
    assert all(valid(s) for s in counts), (path, sorted(counts))
    return sorted(counts), rule


@pytest.mark.parametrize("B", [37, 2731])
@pytest.mark.parametrize("path", ["wg1", "wg2", "wg3", "fc", "box3", "box2"])
def test_split_counts_exact(path, B):
    """wg1: input windows (raw plane); wg2: pixel-pair windows; wg3: the gathered path; fc: the Linear layer (tiled reduce
    at <= 16 splits); box3 / box2: xb_wgrad_box_tc.  Dense at every count, sparse at the rule's."""
    prod, red, units, unit = _launch(path, B)
    counts, rule = _split_counts(path, prod, red, units, unit)
    launches = {n: getattr(tc, n) for n in X.Recorder.NAMES}
    for s in counts:
        for mode in ("dense", "sparse") if s == rule else ("dense",):
            gen = torch.Generator(device=DEV).manual_seed(s)
            X.replay_wgrad(dict(prod, splits=s), dict(red, splits=s), launches, mode, gen, _sm(), tag="B=%d %s: " % (B, path))


@pytest.mark.parametrize("splits,N,C,KH,KW", [
    (1009, 32, 4, 8, 8), (257, 64, 32, 4, 4), (21504, 32, 4, 8, 8), (2, 512, 64, 10, 10), (16, 512, 64, 10, 10),
    (17, 512, 64, 10, 10), (30, 64, 64, 3, 3), (1, 64, 32, 4, 4), (256, 64, 64, 3, 3)])
def test_reduce_order_on_random_partials(splits, N, C, KH, KW):
    """xb_wgrad_reduce (fold, tiled and lane kernels) on random float32 partials of widely spread magnitudes, so that any
    other summation order gives other bits: fresh, scaled by 1/255, and added into an existing gradient."""
    gen = torch.Generator(device=DEV).manual_seed(splits)
    K = C * KH * KW
    p = torch.randn((splits, K, N), generator=gen, device=DEV) * torch.logspace(-8, 8, splits, device=DEV)[:, None, None]
    prev = torch.randn((N, C, KH, KW), generator=gen, device=DEV)
    for scale, acc in ((1.0, False), (1.0 / 255.0, False), (1.0, True), (1.0 / 255.0, True)):
        out = prev.clone() if acc else None
        got = tc.wgrad_reduce(p.clone(), N, C, KH, KW, out=out, accumulate=acc, scale=scale)
        want = X.reduce_ref(p, N, C, KH, KW, scale=scale, out=prev, accumulate=acc, sm_count=_sm())
        X._expect_equal(got, want, "%s splits=%d [%d, %d, %d, %d] scale=%g accumulate=%s"
                        % (X.reduce_kind(splits, N, C, KH, KW), splits, N, C, KH, KW, scale, acc))


@pytest.mark.parametrize("B", [37, 8192])
def test_bias_reduce_order_at_production_row_counts(B):
    """bias_grad's C = KH = KW = 1 form at the column-sum row counts of the plan (conv1 through the halo launch, conv2
    through the box / halo launch of conv3's data gradient, conv3 through the Linear layer's 128-row tiles)."""
    convs, fc = _encoder_modules()
    P = tc.BoxNatureCNN(convs, fc, (84, 84, 4), backend=tc.CudaBackend(3))._plan(B)
    cases = [(P["h_dg2"].m_tiles, 32), (sum(bg.m_tiles for bg, _ in P["dg2"]), 32), (P["dg3"].m_tiles, 64),
             (P["h_dg3"].m_tiles, 64), (-(-B // 128) * 100, 64)]
    gen = torch.Generator(device=DEV).manual_seed(B)
    for rows, N in cases:
        cs = torch.randn((rows, N), generator=gen, device=DEV) * torch.logspace(-6, 6, rows, device=DEV)[:, None]
        prev = torch.randn(N, generator=gen, device=DEV)
        for acc in (False, True):
            got = tc.bias_grad(cs.clone(), N, out=prev.clone() if acc else None, accumulate=acc)
            want = X.reduce_ref(cs.view(-1, 1, N), N, 1, 1, 1, out=prev, accumulate=acc, sm_count=_sm()).view(N)
            X._expect_equal(got, want, "bias rows=%d N=%d accumulate=%s" % (rows, N, acc))


_NO_TMA = r"""
import sys, torch
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import pytest
from xuance_b200.torch.utils import tc_conv as tc
import test_gpu_k12_exact_reductions as T
mp = pytest.MonkeyPatch()
for B in (37, 2731):
    for basic in (False, True):
        T._record_and_replay(mp, T._encoder(basic=basic, cls=tc.TensorCoreNatureCNN), B)
        mp.undo()
for path in ("wg1", "wg2", "wg3", "fc"):
    T.test_split_counts_exact(path, 37)
print("ok")
"""


def test_tma_disabled_in_a_subprocess():
    """XB_K12_TMA=0 (read once by the library): every weight gradient on the cp.async gather - the path the TMA window
    kernels are compared with bit for bit - at production and at every split count above."""
    env = dict(os.environ, XB_K12_TMA="0")
    res = subprocess.run([sys.executable, "-c", _NO_TMA, ROOT], env=env, capture_output=True, text=True, cwd=ROOT)
    assert res.returncode == 0 and "ok" in res.stdout, res.stdout[-4000:] + res.stderr[-4000:]

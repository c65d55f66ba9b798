"""GPU: conv2's data gradient by stride-phase pairs with ReLU masks loaded by bulk copies and g1 rows stored by bulk copies
(conv_tc_kernel_dgrad_phases, taken by xb_gemm_halo_tc for BoxNatureCNN's four 32-column phases into g1's padded layout)
against the generic halo kernel (XB_K12_DGRAD_PHASES=0 in a subprocess), which sums the same products into the same
accumulators in the same order: all three planes of g1 and every column sum must be equal bit for bit, and nothing but
g1's real rows may be written."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
BATCHES = (1, 2, 3, 7, 64, 256, 8192)      # tiles straddling images, a final tile of < 128 positions, the update batch
POISON = 0x5A5A                            # int16 pattern of every element the launch must not write
GUARD = 4096                               # elements after g1

# the reference run: the same inputs through the generic halo kernel only
_REF = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import test_gpu_k12_conv2_dgrad as T
params = torch.load(sys.argv[3])
torch.save({B: [t.cpu() for t in T.run(B, params)] for B in T.BATCHES}, sys.argv[4])
"""


def _plan(B):
    from xuance_b200.torch.utils import tc_conv as tc
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    return tc.BoxNatureCNN(convs, None, (84, 84, 4))._plan(B)


def run(B, params):
    """conv2's data gradient at batch B into a poisoned g1 [3, B * hp1, W1, 32] followed by a guard band; returns the whole
    int16 buffer and the column sums as int32."""
    from xuance_b200.torch.utils import tc_conv as tc
    P = _plan(B)
    hg = P["h_dg2"]
    g = torch.Generator(device=DEV).manual_seed(B)
    g2 = tc.split_bf16(torch.randn(B * P["hp2"], P["W2"], 64, device=DEV, generator=g), 3)
    # act1: plane 0 of both signs, with +0 and -0 (neither passes the ReLU derivative)
    a = torch.randn(B * P["hp1"], P["W1p"], 32, device=DEV, generator=g)
    u = torch.rand(a.shape, device=DEV, generator=g)
    a = torch.where(u < 0.05, torch.zeros_like(a), torch.where(u < 0.1, -torch.zeros_like(a), a))
    act1 = tc.split_bf16(a, 3)
    wd2 = torch.cat([tc.split_bf16(tc.dgrad_weight_matrix(params["w2"].to(DEV), taps), 3) for _, taps in P["dg2"]], 1).contiguous()
    n = 3 * B * P["hp1"] * P["W1"] * 32
    buf = torch.full((n + GUARD,), POISON, dtype=torch.int16, device=DEV)
    g1 = buf[:n].view(torch.bfloat16).view(3, B * P["hp1"], P["W1"], 32)
    cs = torch.full((hg.m_tiles, 32), float("nan"), device=DEV)
    tc.gemm_halo(g2, wd2, hg, out_pl=g1, out_ld=32, relu_mask=act1[0], colsum=cs)
    torch.cuda.synchronize()
    return buf, cs.view(torch.int32)


def _real_rows(B):
    """bool mask of g1's elements that hold real sites (rows off1 .. off1 + H1 - 1 of every image, every pixel)."""
    P = _plan(B)
    m = torch.zeros((3, B, P["hp1"], P["W1"], 32), dtype=torch.bool, device=DEV)
    m[:, :, P["off1"]:P["off1"] + P["H1"]] = True
    return torch.cat([m.view(-1), torch.zeros(GUARD, dtype=torch.bool, device=DEV)])


def _params():
    torch.manual_seed(7)
    return dict(w2=(torch.randn(64, 32, 4, 4) / 8).contiguous())


def test_phase_pair_kernel_is_selected():
    from torch.profiler import ProfilerActivity, profile
    params = _params()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(64, params)
    names = [e.name for e in prof.events() if "conv_tc_kernel" in e.name]
    assert any("conv_tc_kernel_dgrad_phases" in n for n in names), names


def test_g1_and_colsums_bitwise_equal_to_generic_kernel_and_padding_untouched(tmp_path):
    params = _params()
    src, dst = tmp_path / "params.pt", tmp_path / "ref.pt"
    torch.save(params, src)
    env = dict(os.environ, XB_K12_DGRAD_PHASES="0")
    res = subprocess.run([sys.executable, "-c", _REF, ROOT, HERE, str(src), str(dst)], env=env, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    ref = torch.load(dst)
    for B in BATCHES:
        got, cs = run(B, params)
        real = _real_rows(B)
        assert bool((got[~real] == POISON).all()), "B=%d: padding rows or guard band written" % B
        want, want_cs = ref[B][0].to(DEV), ref[B][1].to(DEV)
        assert bool((want[~real] == POISON).all()), "B=%d: the reference wrote outside the real rows" % B
        assert bool((want[real] != POISON).all()), "B=%d: the reference left real elements unwritten" % B
        bad = int((got != want).sum())
        assert bad == 0, "B=%d: %d of %d elements differ" % (B, bad, got.numel())
        bad = int((cs != want_cs).sum())
        assert bad == 0, "B=%d: %d of %d column sums differ" % (B, bad, cs.numel())

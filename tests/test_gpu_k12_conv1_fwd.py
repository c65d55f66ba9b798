"""GPU: conv1's forward from TMA input windows with resident weights and bulk-copied outputs (conv_tc_kernel_fwd_win, taken
by xb_gemm_gather_tc for one raw pixel plane, 4 channels, N = 32, into act1's padded layout) against the gathered cp.async
path (XB_K12_TMA=0 in a subprocess), which sums the same products into the same accumulators in the same order: all three
planes of act1 must be equal bit for bit, and nothing but act1's real sites may be written."""
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
BATCHES = (1, 2, 3, 7, 64, 256, 8192)      # items straddling images, a final item of < 128 sites, the acting batch
POISON = 0x5A5A                            # int16 pattern of every element the launch must not write
GUARD = 4096                               # elements after act1

# the reference run: the same inputs through the gathered path only
_REF = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import test_gpu_k12_conv1_fwd as T
params = torch.load(sys.argv[3])
torch.save({B: T.run(B, params).cpu() for B in T.BATCHES}, sys.argv[4])
"""


def _plan(B):
    from xuance_b200.torch.utils import tc_conv as tc
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2), nn.Conv2d(32, 64, 4, 2, padding=1), nn.Conv2d(64, 64, 3, 1, padding=1)]
    return tc.BoxNatureCNN(convs, None, (84, 84, 4))._plan(B)


def run(B, params):
    """conv1's forward at batch B into a poisoned act1 [3, B * hp1, W1p, 32] followed by a guard band; returns the whole
    int16 buffer."""
    from xuance_b200.torch.utils import tc_conv as tc
    P = _plan(B)
    g = torch.Generator(device=DEV).manual_seed(B)
    x = torch.randint(0, 256, (1, B, 84, 84, 4), device=DEV, generator=g).to(torch.bfloat16)
    n = 3 * B * P["hp1"] * P["W1p"] * 32
    buf = torch.full((n + GUARD,), POISON, dtype=torch.int16, device=DEV)
    act1 = buf[:n].view(torch.bfloat16).view(3, B * P["hp1"], P["W1p"], 32)
    tc.gemm_gather(x, params["w1"].to(DEV), P["fwd1"], bias=params["b1"].to(DEV), relu=True, out_pl=act1, out_ld=32)
    torch.cuda.synchronize()
    return buf


def _real_sites(B):
    """bool mask of act1's elements that hold real sites (rows off1 .. off1 + 20, pixels xo1 .. xo1 + 20 of every image)."""
    P = _plan(B)
    m = torch.zeros((3, B, P["hp1"], P["W1p"], 32), dtype=torch.bool, device=DEV)
    m[:, :, P["off1"]:P["off1"] + P["H1"], P["xo1"]:P["xo1"] + P["W1"]] = True
    return torch.cat([m.view(-1), torch.zeros(GUARD, dtype=torch.bool, device=DEV)])


def _params():
    from xuance_b200.torch.utils import tc_conv as tc
    torch.manual_seed(5)
    w = (torch.randn(32, 4, 8, 8, device=DEV) / 4).contiguous()
    b = torch.randn(32, device=DEV)                               # both signs of the pre-activation: ReLU matters
    return dict(w1=tc.pack_conv_weight(w, 3, 1.0 / 255.0).cpu(), b1=b.cpu())


def test_window_kernel_is_selected():
    from torch.profiler import ProfilerActivity, profile
    params = _params()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(64, params)
    names = [e.name for e in prof.events() if "conv_tc_kernel" in e.name]
    assert any("conv_tc_kernel_fwd_win" in n for n in names), names


def test_act1_bitwise_equal_to_gathered_path_and_padding_untouched(tmp_path):
    params = _params()
    src, dst = tmp_path / "params.pt", tmp_path / "ref.pt"
    torch.save(params, src)
    env = dict(os.environ, XB_K12_TMA="0")
    res = subprocess.run([sys.executable, "-c", _REF, ROOT, HERE, str(src), str(dst)], env=env, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    ref = torch.load(dst)
    for B in BATCHES:
        got = run(B, params)
        real = _real_sites(B)
        assert bool((got[~real] == POISON).all()), "B=%d: padding or guard band written" % B
        want = ref[B].to(DEV)
        assert bool((want[~real] == POISON).all()), "B=%d: the reference wrote outside the real sites" % B
        bad = int((got != want).sum())
        assert bad == 0, "B=%d: %d of %d elements differ" % (B, bad, got.numel())

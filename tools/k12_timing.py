"""Where the K12 warp roles wait (XB_K12_TIMING=1): per layer, mean over CTAs of the clock64 cycles each role spent in its
barrier waits, as a share of the role's lifetime.  Run on a GPU box:  XB_K12_TIMING=1 python tools/k12_timing.py"""
import ctypes, os, sys
os.environ.setdefault("XB_K12_TIMING", "1")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, torch.nn as nn
from xuance_b200 import _lib
from xuance_b200.torch.utils import tc_conv as tc
DEV = "cuda:0"


def report(label, fn):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    fn()
    buf = (ctypes.c_ulonglong * (12 * 132))()
    lib = _lib.load()
    rc = lib.xb_debug_k12_timing(ctypes.addressof(buf), 132)
    assert rc == 0, rc
    t = np.frombuffer(buf, dtype=np.uint64).reshape(132, 12).astype(np.float64)
    m = t.mean(0)
    # consumer warpgroups (wgmma issue + epilogue): slots 0-1, 3; producer warpgroup: slots 4-6 (conv_tc.cu, xb_k12_timing)
    print("%-34s consumer %8.0f clk: wait operands %4.1f%%  wait halo tile %4.1f%% | producer: wait ring %4.1f%%  wait tile buf %4.1f%%"
          % (label, m[0], 100 * m[1] / max(m[0], 1), 100 * m[3] / max(m[0], 1), 100 * m[5] / max(m[4], 1), 100 * m[6] / max(m[4], 1)))


def main():
    B, Pn = int(os.environ.get("XB_K12_BATCH", "8192")), 3
    g = torch.Generator(device=DEV).manual_seed(0)
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2).to(DEV), nn.Conv2d(32, 64, 4, 2, padding=1).to(DEV), nn.Conv2d(64, 64, 3, 1, padding=1).to(DEV)]
    enc = tc.BoxNatureCNN(convs, None, (84, 84, 4), backend=tc.CudaBackend(Pn))
    P = enc._plan(B)
    rnd = lambda *sh: torch.randn(sh, device=DEV, generator=g).to(torch.bfloat16)
    x = torch.randint(0, 256, (1, B, 84, 84, 4), device=DEV, generator=g).to(torch.bfloat16)
    act1, act2 = rnd(Pn, B * P["hp1"], P["W1p"], 32), rnd(Pn, B * P["hp2"], 10, 64)
    act1_pairs = act1.view(Pn, B * P["hp1"], P["W1p"] // 2, 64)
    g3, d2 = rnd(Pn, B * P["hp2"], 10, 64), torch.zeros(Pn, B * P["hp2"], 10, 64, dtype=torch.bfloat16, device=DEV)
    d1 = torch.zeros(Pn, B * P["hp1"], 21, 32, dtype=torch.bfloat16, device=DEV)
    g1 = rnd(Pn, B * P["hp1"] * 21, 32)
    w1 = tc.pack_conv_weight(convs[0].weight.detach(), Pn, 1 / 255.0)
    w2, w3 = tc.pack_conv_weight(convs[1].weight.detach(), Pn), tc.pack_conv_weight(convs[2].weight.detach(), Pn)
    out3 = torch.empty(Pn, B * 100, 64, dtype=torch.bfloat16, device=DEV)
    wd3 = tc.split_bf16(tc.dgrad_weight_matrix(convs[2].weight.detach(), P["taps3"]), Pn)
    wd2 = torch.cat([tc.split_bf16(tc.dgrad_weight_matrix(convs[1].weight.detach(), taps), Pn) for _, taps in P["dg2"]], 1).contiguous()
    report("conv1 forward (gathered cp.async)", lambda: tc.gemm_gather(x, w1, P["fwd1"], relu=True, out_pl=act1, out_ld=32))
    report("conv2 forward (box)", lambda: tc.gemm_box(act1_pairs, w2, P["fwd2"], relu=True, out_pl=d2, out_ld=64))
    report("conv3 forward (box)", lambda: tc.gemm_box(act2, w3, P["fwd3"], relu=True, out_pl=out3, out_ld=64))
    report("conv3 forward (halo)", lambda: tc.gemm_halo(act2, w3, P["h_fwd3"], relu=True, out_pl=out3, out_ld=64))
    report("conv3 data gradient (halo)", lambda: tc.gemm_halo(g3, wd3, P["h_dg3"], out_pl=d2, out_ld=64, relu_mask=act2[0]))
    report("conv2 data gradient (halo)", lambda: tc.gemm_halo(g3, wd2, P["h_dg2"], out_pl=d1, out_ld=32, relu_mask=act1[0]))
    sp = tc.wgrad_box_splits(B * P["hp2"], 6, 576, 64)
    report("conv3 weight gradient (box)", lambda: tc.wgrad_box(act2, g3, P["fwd3"], 6, sp))
    report("conv2 weight gradient (gathered)", lambda: enc.be.wgrad(act1, g3.view(Pn, -1, 64), P["wg2"], 64, 32, 4, 4))
    report("conv1 weight gradient (gathered)", lambda: enc.be.wgrad(x, g1, P["wg1"], 32, 4, 8, 8))
    # the Linear layer 6400 -> 512
    xf, wf = rnd(Pn, B, 6400), rnd(Pn, 512, 6400)
    yf = torch.empty(Pn, B, 512, dtype=torch.bfloat16, device=DEV)
    report("Linear forward (TMA tiles)", lambda: tc.gemm_gather(xf, wf, tc.linear_geometry(B, 6400), relu=True, out_pl=yf))


if __name__ == "__main__":
    main()

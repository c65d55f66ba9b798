"""K12 on the GPU, two reports.

    XB_K12_TIMING=1 python tools/k12_timing.py             where the warp roles wait (default mode)
    XB_K12_TIMING=0 python tools/k12_timing.py --launches  CUDA-event time of every K12 launch of one encoder update

Role timing: per layer, mean over CTAs of the clock64 cycles each role spent in its barrier waits, as a share of the
role's lifetime.  Per-launch table: BoxNatureCNN's real plan at B = 8192 (XB_K12_BATCH), three planes, raw uint8 pixels,
one forward + backward of conv1-3 and the 6400 -> 512 layer exactly as an update runs them; each launch gets its own label
(conv3's forward and data gradient have the same GEMM shape), the median over the timed repetitions, and the executed
bf16 TFLOP/s of tc_conv's FLOP log.  ``--json PATH`` also writes the table."""
import argparse, ctypes, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
DEV = "cuda:0"


def report(label, fn):
    import numpy as np, torch
    from xuance_b200 import _lib
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
    # consumer warpgroups (wgmma issue + epilogue): slots 0-3, 7; producer warpgroup: slots 4-6 (conv_tc.cu, xb_k12_timing)
    c = lambda s: 100 * m[s] / max(m[0], 1)
    print("%-34s consumer %8.0f clk: wait operands %4.1f%%  wait halo tile %4.1f%%  wgmma wait %4.1f%%  epilogue %4.1f%% | "
          "producer: wait ring %4.1f%%  wait tile buf %4.1f%%"
          % (label, m[0], c(1), c(3), c(2), c(7), 100 * m[5] / max(m[4], 1), 100 * m[6] / max(m[4], 1)))


def roles():
    import torch, torch.nn as nn
    from xuance_b200.torch.utils import tc_conv as tc
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
    report("conv1 forward (TMA windows)", lambda: tc.gemm_gather(x, w1, P["fwd1"], relu=True, out_pl=act1, out_ld=32))
    report("conv2 forward (box)", lambda: tc.gemm_box(act1_pairs, w2, P["fwd2"], relu=True, out_pl=d2, out_ld=64))
    report("conv3 forward (box)", lambda: tc.gemm_box(act2, w3, P["fwd3"], relu=True, out_pl=out3, out_ld=64))
    report("conv3 forward (halo)", lambda: tc.gemm_halo(act2, w3, P["h_fwd3"], relu=True, out_pl=out3, out_ld=64))
    report("conv3 data gradient (halo)", lambda: tc.gemm_halo(g3, wd3, P["h_dg3"], out_pl=d2, out_ld=64, relu_mask=act2[0]))
    cs1 = torch.empty(P["h_dg2"].m_tiles, 32, device=DEV)
    report("conv2 data gradient (phase pairs)", lambda: tc.gemm_halo(g3, wd2, P["h_dg2"], out_pl=d1, out_ld=32, relu_mask=act1[0], colsum=cs1))
    sp = tc.wgrad_box_splits(B * P["hp2"], 6, 576, 64)
    report("conv3 weight gradient (box)", lambda: tc.wgrad_box(act2, g3, P["fwd3"], 6, sp))
    report("conv2 weight gradient (TMA pairs)", lambda: enc.be.wgrad(act1, g3.view(Pn, -1, 64), P["wg2"], 64, 32, 4, 4))
    report("conv1 weight gradient (TMA windows)", lambda: enc.be.wgrad(x, g1, P["wg1"], 32, 4, 8, 8))
    # the Linear layer 6400 -> 512
    xf, wf = rnd(Pn, B, 6400), rnd(Pn, 512, 6400)
    yf = torch.empty(Pn, B, 512, dtype=torch.bfloat16, device=DEV)
    report("Linear forward (TMA tiles)", lambda: tc.gemm_gather(xf, wf, tc.linear_geometry(B, 6400), relu=True, out_pl=yf))


def launch_labels(tc, P):
    """(ABI name, label) of every K12 launch of BoxNatureCNN.forward + backward, in launch order (tc_conv.py)."""
    dg = "xb_gemm_halo_tc" if tc.HALO3 else "xb_gemm_box_tc"
    wg = lambda box: "xb_wgrad_box_tc" if box else "xb_wgrad_gather_tc"
    seq = [("xb_gemm_gather_tc", "conv1 forward (TMA windows)"), ("xb_gemm_box_tc", "conv2 forward"), (dg, "conv3 forward"),
           ("xb_gemm_gather_tc", "Linear forward"), ("xb_wgrad_gather_tc", "Linear weight gradient"),
           ("xb_gemm_gather_tc", "Linear data gradient"), (wg(tc.BOX_WGRAD3), "conv3 weight gradient"),
           (dg, "conv3 data gradient"), (wg(tc.BOX_WGRAD2), "conv2 weight gradient")]
    if tc.HALO and P["h_dg2"] is not None:
        seq.append(("xb_gemm_halo_tc", "conv2 data gradient (phase pairs)"))
    else:
        seq += [("xb_gemm_box_tc", "conv2 data gradient, phase %d" % i) for i in range(len(P["dg2"]))]
    return seq + [("xb_wgrad_gather_tc", "conv1 weight gradient")]


def launches(reps, json_path):
    import numpy as np, torch, torch.nn as nn
    from xuance_b200 import _lib
    from xuance_b200.torch.utils import tc_conv as tc
    B = int(os.environ.get("XB_K12_BATCH", "8192"))
    torch.manual_seed(0)
    convs = [nn.Conv2d(4, 32, 8, 4, padding=2).to(DEV), nn.Conv2d(32, 64, 4, 2, padding=1).to(DEV), nn.Conv2d(64, 64, 3, 1, padding=1).to(DEV)]
    fc = nn.Linear(6400, 512).to(DEV)
    enc = tc.BoxNatureCNN(convs, fc, (84, 84, 4), backend=tc.CudaBackend(3))
    P = enc._plan(B)
    x = torch.randint(0, 256, (1, B, 84, 84, 4), device=DEV).to(torch.bfloat16)
    dz = torch.randn(B, 512, device=DEV) * 1e-3
    names = sorted({n for n, _ in launch_labels(tc, P)})

    def update():
        enc.forward(x, B)
        enc.backward(dz)
    update()
    torch.cuda.synchronize()
    times, log = [], None
    for _ in range(reps):
        _lib.profile, tc.flop_log = {n: [] for n in names}, []
        update()
        torch.cuda.synchronize()
        prof, log = _lib.profile, tc.flop_log
        _lib.profile, tc.flop_log = None, None
        it = {n: iter(prof[n]) for n in names}
        times.append([(lambda ab: ab[0].elapsed_time(ab[1]))(next(it[nm])) for nm, _, _, _ in log])
    seq = launch_labels(tc, P)
    assert [nm for nm, _, _, _ in log] == [n for n, _ in seq], ([nm for nm, *_ in log], seq)
    ms = np.median(np.array(times), 0)
    props = torch.cuda.get_device_properties(0)
    rows = []
    for (nm, label), (_, tag, fl, _), t in zip(seq, log, ms):
        rows.append(dict(label=label, abi=nm, shape=tag, ms=float(t), tflops_executed=fl / (t * 1e-3) / 1e12))
        print("%-34s %-20s %-40s %7.3f ms  %6.1f TFLOP/s" % (label, nm, tag, t, rows[-1]["tflops_executed"]))
    total = float(ms.sum())
    print("%-34s %69.3f ms  (B = %d, %s, XB_K12_HALO=%s XB_K12_BOX_WGRAD=%s)" % ("sum", total, B, props.name, tc.HALO_MODE, tc.BOX_WGRAD))
    if json_path:
        with open(json_path, "w") as fh:
            json.dump(dict(device=props.name, batch=B, halo=tc.HALO_MODE, box_wgrad=tc.BOX_WGRAD, reps=reps, sum_ms=total,
                           launches=rows), fh, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", action="store_true", help="per-launch CUDA-event table instead of the role timing")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if a.launches:
        os.environ["XB_K12_TIMING"] = "0"        # the role clocks cost time inside the kernel
        launches(a.reps, a.json)
    else:
        os.environ.setdefault("XB_K12_TIMING", "1")
        roles()


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Per-kernel roofline numbers for every entry point of include/xb200.h, at the BASELINE shapes and at HBM-sized
shapes (SURVEY.md section 7 "hard parts": at the named PPO shape K2/K4/K5 move < 1 MB and are launch-bound, so the
bandwidth fraction is also reported at a scaled shape).  CUDA events on the launching stream, >= 3 warm-ups, L2
flushed between timed launches (256 MB memset).  Prints one JSON object.

    python tools/kernel_bench.py [--only k2,k4] [--reps 20]      (k12 / k12box / k3p: the tensor-core encoder layers, gathered and TMA-box / halo variants; k13: the GRU sequence kernels against cuDNN; k13l: the LSTM sequence kernels against cuDNN)
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from xuance_b200 import _lib  # noqa: E402

DEV = torch.device("cuda:0")


def peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return float(d["hbm_gbs"]), float(d.get("bf16_tflops", 1590.0)), "measured"
    return 6650.0, 1590.0, "fallback"


_flush = None


def timeit(fn, reps, flush=True):
    global _flush
    if _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        if flush:
            _flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    return float(np.median(ts))


def entry(name, shape, us, alg_bytes, hbm, flops=None, tpeak=None):
    d = {"kernel": name, "shape": shape, "us": round(us, 2), "algorithmic_bytes": int(alg_bytes),
         "GBps": round(alg_bytes / us / 1e3, 1), "frac_hbm": round(alg_bytes / us / 1e3 / hbm, 3)}
    if flops:
        d["TFLOPs"] = round(flops / us / 1e6, 2)
        d["frac_bf16_peak"] = round(flops / us / 1e6 / tpeak, 4)
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--small", action="store_true", help="skip the 100M-element optimiser case (profiling runs)")
    args = ap.parse_args()
    only = set(x for x in args.only.split(",") if x)
    want = lambda k: not only or k in only
    hbm, tpk, src = peak()
    out = {"hbm_peak_GBps": hbm, "bf16_peak_TFLOPs": tpk, "peak_source": src, "kernels": []}
    add = out["kernels"].append
    g = torch.Generator(device=DEV).manual_seed(0)
    R = args.reps

    if want("k1"):
        N, T, rb = 256, 128, 28224
        buf = torch.zeros((N, T, rb), dtype=torch.uint8, device=DEV)
        src_rows = torch.randint(0, 256, (N, rb), dtype=torch.uint8, device=DEV, generator=g)
        fields = torch.zeros((5, N, T), device=DEV)
        scal = torch.randn((5, N), device=DEV)
        us = timeit(lambda: _lib.call("xb_rollout_store", _lib.ptr(buf), _lib.ptr(src_rows), rb, _lib.ptr(fields),
                                      _lib.ptr(scal), 5, N, T, 7), R)
        add(entry("K1 xb_rollout_store", "256 envs x 28224 B + 5 fields", us, 2 * N * (rb + 20), hbm))
        del buf

    if want("k2"):
        for N, T in ((256, 128), (4096, 1024)):
            rew, val = torch.randn((N, T), device=DEV), torch.randn((N, T), device=DEV)
            term = (torch.rand((N, T), device=DEV) < 0.01).float()
            seg = torch.zeros((N, T), dtype=torch.uint8, device=DEV)
            seg[:, -1] = 1
            boot = torch.randn((N, T), device=DEV)
            cov = torch.full((N,), T, dtype=torch.int32, device=DEV)
            adv, ret = torch.empty((N, T), device=DEV), torch.empty((N, T), device=DEV)
            us = timeit(lambda: _lib.call("xb_gae_scan", _lib.ptr(rew), _lib.ptr(val), _lib.ptr(term), _lib.ptr(seg),
                                          _lib.ptr(boot), _lib.ptr(cov), _lib.ptr(adv), _lib.ptr(ret), N, T, 0.99, 0.95, 1), R)
            add(entry("K2 xb_gae_scan", f"{N} envs x {T} steps", us, 21 * N * T + 8 * N, hbm))

    if want("k3"):
        S, B, H, W, C = 256 * 128, 8192, 84, 84, 4
        rb = H * W * C
        src_obs = torch.randint(0, 256, (S, rb), dtype=torch.uint8, device=DEV, generator=g)
        idx = torch.randperm(S, device=DEV, generator=g)[:B].contiguous()
        dst = torch.empty((B, rb), dtype=torch.uint8, device=DEV)
        us = timeit(lambda: _lib.call("xb_gather_rows", _lib.ptr(src_obs), _lib.ptr(idx), B, rb, _lib.ptr(dst)), R)
        add(entry("K3 xb_gather_rows (u8, bulk-async)", "8192 rows x 28224 B", us, 2 * B * rb + 8 * B, hbm))
        for fmt, name, w, dt in ((_lib.OBS_F32_NCHW, "f32 NCHW", 4, torch.float32), (_lib.OBS_F32_NHWC, "f32 NHWC", 4, torch.float32),
                                 (_lib.OBS_BF16_NHWC, "bf16 NHWC", 2, torch.bfloat16)):
            o = torch.empty((B, rb), dtype=dt, device=DEV)
            us = timeit(lambda: _lib.call("xb_gather_obs", _lib.ptr(src_obs), _lib.ptr(idx), B, H, W, C, _lib.ptr(o), fmt), R)
            add(entry(f"K3 xb_gather_obs ({name})", "8192 rows x 28224 px", us, B * rb * (1 + w) + 8 * B, hbm))
            del o
        del src_obs, dst
        for slots, Bs in ((256 * 128, 8192), (1 << 24, 1 << 22)):
            F = 5
            fields = torch.randn((F, slots), device=DEV)
            idx = torch.randint(0, slots, (Bs,), device=DEV, generator=g)
            o = torch.empty((F, Bs), device=DEV)
            stats, scratch = torch.zeros(2, device=DEV), _lib.scratch(DEV)
            us = timeit(lambda: _lib.call("xb_gather_scalars", _lib.ptr(fields), slots, _lib.ptr(idx), Bs, F, _lib.ptr(o),
                                          4, _lib.ptr(stats), _lib.ptr(scratch)), R)
            add(entry("K3 xb_gather_scalars (+adv norm, 2 launches)", f"{Bs} of {slots} slots x 5 fields", us,
                      Bs * (8 + 4 * F * 2 + 8), hbm))

    if want("k4"):
        for B in (8192, 1 << 22):
            A = 4
            lg, v = torch.randn((B, A), device=DEV), torch.randn(B, device=DEV)
            act = torch.randint(0, A, (B,), device=DEV).float()
            old, adv, ret = torch.randn(B, device=DEV) * 0.1 - 1.4, torch.randn(B, device=DEV), torch.randn(B, device=DEV)
            dl, dv = torch.empty((B, A), device=DEV), torch.empty(B, device=DEV)
            stats, scratch = torch.zeros(8, device=DEV), _lib.scratch(DEV)
            us = timeit(lambda: _lib.call("xb_ppo_loss_fwd_bwd", _lib.ptr(lg), _lib.ptr(v), _lib.ptr(act), _lib.ptr(old),
                                          _lib.ptr(adv), _lib.ptr(ret), B, A, B, 0.2, 0.25, 0.01, 0, _lib.ptr(dl), _lib.ptr(dv),
                                          _lib.ptr(stats), _lib.ptr(scratch)), R)
            add(entry("K4 xb_ppo_loss_fwd_bwd", f"B={B}, A=4", us, B * 56, hbm))

    if want("k6z"):
        # C51 / QR-DQN at the config shapes: CartPole (B=256, A=2), SyntheticAtari (B=32, A=4), full ALE set (A=18).
        # Algorithmic bytes per row: greedy 4*A*N in + 8 out; losses 8*A*N in (eval + target rows) + 12 scalars in,
        # 4*A*N gradient + 8 target action out.
        for B, A in ((256, 2), (32, 4), (32, 18)):
            for algo, N in (("c51", 51), ("qrdqn", 20)):
                z, zn = torch.randn((B, A, N), device=DEV), torch.randn((B, A, N), device=DEV)
                sup = torch.linspace(-10, 10, N).to(DEV) if algo == "c51" else None
                act = torch.randint(0, A, (B,), device=DEV).float()
                rew, ter = torch.randn(B, device=DEV), (torch.rand(B, device=DEV) < 0.1).float()
                grad, ga = torch.empty_like(z), torch.empty(B, dtype=torch.int64, device=DEV)
                stats, scratch = torch.zeros(4, device=DEV), _lib.scratch(DEV)
                us = timeit(lambda: _lib.call("xb_dist_greedy", _lib.ptr(z), _lib.ptr(sup), B, A, N, _lib.ptr(ga), None,
                                              None), R)
                add(entry("K6Z xb_dist_greedy (%s)" % algo, f"B={B}, A={A}, N={N}", us, B * (4 * A * N + 8), hbm))
                if algo == "c51":
                    fn = lambda: _lib.call("xb_c51_loss_fwd_bwd", _lib.ptr(z), _lib.ptr(zn), _lib.ptr(sup), _lib.ptr(act),
                                           _lib.ptr(rew), _lib.ptr(ter), B, A, N, B, 0.99, -10.0, 10.0, 0.4,
                                           _lib.ptr(grad), _lib.ptr(ga), None, _lib.ptr(stats), _lib.ptr(scratch))
                else:
                    fn = lambda: _lib.call("xb_qrdqn_loss_fwd_bwd", _lib.ptr(z), _lib.ptr(zn), _lib.ptr(act),
                                           _lib.ptr(rew), _lib.ptr(ter), B, A, N, B, 0.99, _lib.ptr(grad), _lib.ptr(ga),
                                           _lib.ptr(stats), _lib.ptr(scratch))
                us = timeit(fn, R)
                add(entry("K6Z xb_%s_loss_fwd_bwd" % algo, f"B={B}, A={A}, N={N}", us, B * (12 * A * N + 20), hbm))

    if want("k5"):
        N, cap, B = 16, 65536, 512
        k = B // N
        st = torch.rand((N, 2 * cap), device=DEV)
        mt = torch.rand((N, 2 * cap), device=DEV)
        mp = torch.ones(N, device=DEV)
        u = torch.rand((N, k), device=DEV)
        so, fo = torch.empty((N, k), dtype=torch.int64, device=DEV), torch.empty(N * k, dtype=torch.int64, device=DEV)
        wo = torch.empty((N, k), dtype=torch.float64, device=DEV)
        lvl = cap // 2
        while lvl >= 1:
            st[:, lvl:2 * lvl] = st[:, 2 * lvl:4 * lvl:2] + st[:, 2 * lvl + 1:4 * lvl:2]
            lvl //= 2
        us = timeit(lambda: _lib.call("xb_per_sample", _lib.ptr(st), _lib.ptr(mt), _lib.ptr(u), N, cap, cap, k, cap, 0.01,
                                      _lib.ptr(so), _lib.ptr(fo), _lib.ptr(wo)), R, flush=False)
        add(entry("K5 xb_per_sample (L2-resident trees)", "16 envs x 65536 leaves, B=512", us, B * (17 * 4 + 24), hbm))
        pr = torch.rand(B, device=DEV)
        us = timeit(lambda: _lib.call("xb_per_update", _lib.ptr(st), _lib.ptr(mt), _lib.ptr(mp), _lib.ptr(so), _lib.ptr(pr),
                                      N, cap, k, 0.5), R, flush=False)
        add(entry("K5 xb_per_update", "16 envs x 65536 leaves, B=512", us, B * 2 * 16 * 12, hbm))
        us = timeit(lambda: _lib.call("xb_per_insert", _lib.ptr(st), _lib.ptr(mt), _lib.ptr(mp), N, cap, 123, 0.5), R, flush=False)
        add(entry("K5 xb_per_insert", "16 envs", us, N * 2 * 16 * 12, hbm))

    if want("k6"):
        for B in (512, 1 << 22):
            A = 6
            qe, qn = torch.randn((B, A), device=DEV), torch.randn((B, A), device=DEV)
            act = torch.randint(0, A, (B,), device=DEV).float()
            rew, ter = torch.randn(B, device=DEV), (torch.rand(B, device=DEV) < 0.1).float()
            dq, td = torch.empty((B, A), device=DEV), torch.empty(B, device=DEV)
            stats, scratch = torch.zeros(4, device=DEV), _lib.scratch(DEV)
            us = timeit(lambda: _lib.call("xb_dqn_td_fwd_bwd", _lib.ptr(qe), _lib.ptr(qn), None, _lib.ptr(act), _lib.ptr(rew),
                                          _lib.ptr(ter), B, A, B, 0.99, _lib.ptr(dq), _lib.ptr(td), _lib.ptr(stats),
                                          _lib.ptr(scratch)), R)
            add(entry("K6 xb_dqn_td_fwd_bwd", f"B={B}, A=6", us, B * ((2 * A + 3) * 4 + (A + 1) * 4), hbm))

    if want("k7"):
        for n in ((3358887,) if args.small else (3358887, 100_000_000)):
            n = (n + 31) // 32 * 32
            p, gr = torch.randn(n, device=DEV), torch.randn(n, device=DEV)
            m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
            hyper, norm, scratch = torch.tensor([1e-4, 0.03, 0, 0], device=DEV), torch.zeros(1, device=DEV), _lib.scratch(DEV)
            us = timeit(lambda: _lib.call("xb_grad_sumsq", _lib.ptr(gr), n, 1.0, _lib.ptr(norm), _lib.ptr(scratch)), R)
            add(entry("K7 xb_grad_sumsq", f"n={n}", us, 4 * n, hbm))
            us = timeit(lambda: _lib.call("xb_adam_step", _lib.ptr(p), _lib.ptr(gr), _lib.ptr(m), _lib.ptr(v), n, _lib.ptr(hyper),
                                          0.9, 0.999, 1e-5, 0.5, _lib.ptr(norm), 1.0, 0), R)
            add(entry("K7 xb_adam_step", f"n={n}", us, 28 * n, hbm))
            del p, gr, m, v

    if want("k9"):
        from xuance_b200.torch.rl_models import QMIX_Mixer
        n, S, H = 5, 98, 32
        mixer = QMIX_Mixer(S, 32, 32, n, "cuda:0")
        for Rr in (1920, 245760):
            q, w1 = torch.randn((Rr, n), device=DEV), torch.randn((Rr, n * H), device=DEV)
            b1, w2, b2 = torch.randn((Rr, H), device=DEV), torch.randn((Rr, H), device=DEV), torch.randn(Rr, device=DEV)
            y = torch.empty(Rr, device=DEV)
            us = timeit(lambda: _lib.call("xb_qmix_mix_fwd", _lib.ptr(q), _lib.ptr(w1), _lib.ptr(b1), _lib.ptr(w2), _lib.ptr(b2),
                                          Rr, n, H, _lib.ptr(y)), R)
            add(entry("K9 xb_qmix_mix_fwd (epilogue only)", f"{Rr} rows", us, Rr * (n * H + 2 * H + n + 2) * 4, hbm))
            dy = torch.randn(Rr, device=DEV)
            dq, dw1, db1, dw2 = torch.empty_like(q), torch.empty_like(w1), torch.empty_like(b1), torch.empty_like(w2)
            us = timeit(lambda: _lib.call("xb_qmix_mix_bwd", _lib.ptr(dy), _lib.ptr(q), _lib.ptr(w1), _lib.ptr(b1), _lib.ptr(w2),
                                          Rr, n, H, _lib.ptr(dq), _lib.ptr(dw1), _lib.ptr(db1), _lib.ptr(dw2)), R)
            add(entry("K9 xb_qmix_mix_bwd", f"{Rr} rows", us, Rr * ((n * H + 2 * H + n + 1) * 4 + (n * H + 2 * H + n) * 4), hbm))
            st = torch.randn((Rr, S), device=DEV)
            flops = Rr * 2.0 * (S * 128 + 32 * (n * H + H + 1))
            with torch.no_grad():
                mixer.use_tensor_core_forward = True
                us_tc = timeit(lambda: mixer(q, st), R)
                mixer.use_tensor_core_forward = False
                us_lib = timeit(lambda: mixer(q, st), R)
            e = entry("K9-TC xb_qmix_mix_fused_fwd (wgmma, incl. torch.cat of weights)", f"{Rr} rows, S=98, n=5", us_tc,
                      Rr * (S + n + 1) * 4, hbm, flops, tpk)
            e["vs_cublas_plus_epilogue_us"] = round(us_lib, 2)
            add(e)

    if want("k10"):
        for N, A in ((256, 4), (1 << 20, 4), (1 << 20, 18)):
            logits = torch.randn((N, A), device=DEV, generator=g)
            u = torch.rand(N, device=DEV, generator=g)
            af, ai, lp = torch.empty(N, device=DEV), torch.empty(N, dtype=torch.int32, device=DEV), torch.empty(N, device=DEV)
            us = timeit(lambda: _lib.call("xb_categorical_act", _lib.ptr(logits), _lib.ptr(u), None, N, A, _lib.ptr(af),
                                          _lib.ptr(ai), _lib.ptr(lp), None), R)
            add(entry("K10 xb_categorical_act", f"{N}x{A}", us, N * ((A + 1) * 4 + 12), hbm))

    if want("k11"):
        for N, D in ((8, 4), (256, 28224), (256, 1 << 20)):
            x = torch.randn((N, D), device=DEV, generator=g)
            mean, var, y = torch.zeros(D, device=DEV), torch.ones(D, device=DEV), torch.empty_like(x)
            us = timeit(lambda: _lib.call("xb_rms_update_normalize", _lib.ptr(x), N, D, _lib.ptr(mean), _lib.ptr(var), 1e-4, 1,
                                          _lib.ptr(y), 5.0, 1e-8), R)
            add(entry("K11 xb_rms_update_normalize", f"{N}x{D}", us, N * D * 4 * 2, hbm))     # one read + one write (algorithmic)

    if want("k3p"):
        from xuance_b200 import _lib as L
        Nn, T, rb, B = 256, 128, 28224, 8192
        buf = torch.randint(0, 256, (Nn * T, rb), dtype=torch.uint8, device=DEV, generator=g)
        idx = torch.randperm(Nn * T, device=DEV, generator=g)[:B].contiguous()
        for P in (1, 2, 3):
            dst = torch.empty((P, B, rb), dtype=torch.bfloat16, device=DEV)
            us = timeit(lambda: L.call("xb_gather_obs_planes", L.ptr(buf), L.ptr(idx), B, rb, P, L.ptr(dst)), R)
            add(entry(f"K3-P xb_gather_obs_planes (P={P})", f"{B} rows x {rb} B", us, B * rb * (1 + 2 * P) + 8 * B, hbm))

    if want("k12"):
        # tensor-core layers at the PPO minibatch (8192 samples): forward, data gradient, weight gradient.
        # flops = fp32-equivalent 2*M*N*K of the layer (the tensor pipe executes 3x / 6x that in bf16 MMAs; conv1 reads ONE
        # exact plane of raw pixels, so its factor is 2 / 3)
        from xuance_b200.torch.utils import tc_conv as tc
        B = int(os.environ.get("XB_K12_BATCH", "8192"))
        layers = (("conv1", 84, 84, 4, 32, 8, 4), ("conv2", 21, 21, 32, 64, 4, 2), ("conv3", 10, 10, 64, 64, 3, 1))
        for P in (3, 2):
            for name, H, W, C, N, k, s in layers:
                pad = (k - s) // 2
                geom = tc.conv_forward_geometry(B, H, W, C, k, k, s, pad)
                w = torch.randn((N, C, k, k), device=DEV, generator=g) / np.sqrt(C * k * k)
                if name == "conv1":
                    x_pl = torch.randint(0, 256, (1, B, H, W, C), device=DEV, generator=g).to(torch.bfloat16)
                    w_pl = tc.pack_conv_weight(w, P, 1.0 / 255.0)
                else:
                    x_pl = tc.split_bf16(torch.rand((B, H, W, C), device=DEV, generator=g), P)
                    w_pl = tc.pack_conv_weight(w, P)
                out_pl = torch.empty((P, geom.M, N), dtype=torch.bfloat16, device=DEV)
                fl = 2.0 * geom.M * N * geom.K
                byts = x_pl.numel() * 2 + w_pl.numel() * 2 + out_pl.numel() * 2
                us = timeit(lambda: tc.gemm_gather(x_pl, w_pl, geom, relu=True, out_pl=out_pl), R)
                add(entry(f"K12 forward {name} (PA={x_pl.shape[0]} PB={P})", f"M={geom.M} N={N} K={geom.K}", us, byts, hbm, fl, tpk))
                g_pl = tc.split_bf16(torch.randn((geom.M, N), device=DEV, generator=g), P)
                splits = tc.wgrad_splits(geom.M, geom.K)
                us = timeit(lambda: tc.wgrad_reduce(tc.wgrad_gather(x_pl, g_pl, geom, splits), N, C, k, k), R)
                add(entry(f"K12 weight gradient {name} (PA={x_pl.shape[0]} PB={P}, {splits} splits)", f"M={geom.M} N={N} K={geom.K}", us,
                          x_pl.numel() * 2 + g_pl.numel() * 2, hbm, fl, tpk))
                if name != "conv1":
                    phases = tc.conv_dgrad_geometries(B, H, W, C, k, k, s, pad, N)
                    wds = [tc.split_bf16(tc.dgrad_weight_matrix(w, taps), P) for _, taps in phases]
                    dx_pl = torch.empty((P, B * H * W, C), dtype=torch.bfloat16, device=DEV)

                    def run_dgrad():
                        for (gm, _), wd in zip(phases, wds):
                            tc.gemm_gather(g_pl, wd, gm, out_pl=dx_pl, out_ld=C, relu_mask=x_pl[0].reshape(-1, C))
                    us = timeit(run_dgrad, R)
                    add(entry(f"K12 data gradient {name} (P={P}, {len(phases)} phases)", f"M={B * H * W} N={C}", us,
                              g_pl.numel() * 2 + dx_pl.numel() * 2, hbm, fl, tpk))
                del x_pl, w_pl, out_pl, g_pl
            # the hidden layer 6400 -> 512: forward, data gradient, weight gradient (column tiles inside one launch)
            geom = tc.linear_geometry(B, 6400)
            x_pl = tc.split_bf16(torch.rand((B, 6400), device=DEV, generator=g), P)
            wf = torch.randn((512, 6400), device=DEV, generator=g) / 80.0
            w_pl = tc.split_bf16(wf, P)
            out_fc = torch.empty((B, 512), device=DEV)
            fl = 2.0 * B * 512 * 6400
            us = timeit(lambda: tc.gemm_gather(x_pl, w_pl, geom, relu=True, out_f32=out_fc), R)
            add(entry(f"K12 forward fc 6400->512 (P={P})", f"M={B} N=512 K=6400", us,
                      x_pl.numel() * 2 + w_pl.numel() * 2 + out_fc.numel() * 4, hbm, fl, tpk))
            g_pl = tc.split_bf16(torch.randn((B, 512), device=DEV, generator=g), P)
            wt_pl = tc.split_bf16(wf.t().contiguous(), P)
            dx_pl = torch.empty((P, B, 6400), dtype=torch.bfloat16, device=DEV)
            us = timeit(lambda: tc.gemm_gather(g_pl, wt_pl, tc.linear_geometry(B, 512), out_pl=dx_pl, relu_mask=x_pl[0]), R)
            add(entry(f"K12 data gradient fc (P={P})", f"M={B} N=6400 K=512", us,
                      g_pl.numel() * 2 + wt_pl.numel() * 2 + dx_pl.numel() * 2, hbm, fl, tpk))
            nt = 512 // tc.n_tile_for(512, P)
            splits = tc.wgrad_splits(B, 6400, nt)
            us = timeit(lambda: tc.wgrad_reduce(tc.wgrad_gather(x_pl, g_pl, geom, splits), 512, 6400, 1, 1), R)
            add(entry(f"K12 weight gradient fc (P={P}, {splits} splits)", f"M={B} N=512 K=6400", us,
                      x_pl.numel() * 2 + g_pl.numel() * 2 + 512 * 6400 * 4, hbm, fl, tpk))
            del x_pl, w_pl, g_pl, wt_pl, dx_pl
    if want("k12box"):
        # the convolutions after the first with padded-row activations + TMA boxes (BoxNatureCNN's geometries), 3 planes
        import torch.nn as nn
        from xuance_b200.torch.utils import tc_conv as tc
        B, Pn = int(os.environ.get("XB_K12_BATCH", "8192")), 3
        convs = [nn.Conv2d(4, 32, 8, 4, padding=2).to(DEV), nn.Conv2d(32, 64, 4, 2, padding=1).to(DEV), nn.Conv2d(64, 64, 3, 1, padding=1).to(DEV)]
        enc = tc.BoxNatureCNN(convs, None, (84, 84, 4), backend=tc.CudaBackend(Pn))
        P = enc._plan(B)
        rnd = lambda *sh: torch.randn(sh, device=DEV, generator=g).to(torch.bfloat16)
        act1, act2 = rnd(Pn, B * P["hp1"], P["W1p"], 32), rnd(Pn, B * P["hp2"], 10, 64)
        act1_pairs = act1.view(Pn, B * P["hp1"], P["W1p"] // 2, 64)
        g3, d2, d1 = rnd(Pn, B * P["hp2"], 10, 64), torch.zeros(Pn, B * P["hp2"], 10, 64, dtype=torch.bfloat16, device=DEV), torch.zeros(Pn, B * P["hp1"], 21, 32, dtype=torch.bfloat16, device=DEV)
        w2, w3 = tc.pack_conv_weight(convs[1].weight.detach(), Pn), tc.pack_conv_weight(convs[2].weight.detach(), Pn)
        out3 = torch.empty(Pn, B * 100, 64, dtype=torch.bfloat16, device=DEV)
        us = timeit(lambda: tc.gemm_box(act1_pairs, w2, P["fwd2"], relu=True, out_pl=d2, out_ld=64), R)
        add(entry("K12-box forward conv2 (P=3)", f"M={B * 100} N=64 K=512", us, act1.numel() * 2 + d2.numel() * 2, hbm, 2.0 * B * 100 * 64 * 512, tpk))
        us = timeit(lambda: tc.gemm_box(act2, w3, P["fwd3"], relu=True, out_pl=out3, out_ld=64), R)
        add(entry("K12-box forward conv3 (P=3)", f"M={B * 100} N=64 K=576", us, act2.numel() * 2 + out3.numel() * 2, hbm, 2.0 * B * 100 * 64 * 576, tpk))
        wd3 = tc.split_bf16(tc.dgrad_weight_matrix(convs[2].weight.detach(), P["taps3"]), Pn)
        us = timeit(lambda: tc.gemm_box(g3, wd3, P["dg3"], out_pl=d2, out_ld=64, relu_mask=act2[0]), R)
        add(entry("K12-box data gradient conv3 (P=3)", f"M={B * 100} N=64 K=576", us, g3.numel() * 2 + d2.numel() * 2, hbm, 2.0 * B * 100 * 64 * 576, tpk))
        wds = [tc.split_bf16(tc.dgrad_weight_matrix(convs[1].weight.detach(), taps), Pn) for _, taps in P["dg2"]]

        def run_dg2():
            for (bg, _), wd in zip(P["dg2"], wds):
                tc.gemm_box(g3, wd, bg, out_pl=d1, out_ld=32, relu_mask=act1[0])
        us = timeit(run_dg2, R)
        add(entry("K12-box data gradient conv2 (P=3, 4 phases)", f"M={B * 441} N=32 K=256", us, 4 * g3.numel() * 2 + d1.numel() * 2, hbm, 2.0 * B * 100 * 64 * 512, tpk))
        us = timeit(lambda: tc.gemm_halo(act2, w3, P["h_fwd3"], relu=True, out_pl=out3, out_ld=64), R)
        add(entry("K12-halo forward conv3 (P=3)", f"M={B * 100} N=64 K=576", us, act2.numel() * 2 + out3.numel() * 2, hbm, 2.0 * B * 100 * 64 * 576, tpk))
        us = timeit(lambda: tc.gemm_halo(g3, wd3, P["h_dg3"], out_pl=d2, out_ld=64, relu_mask=act2[0]), R)
        add(entry("K12-halo data gradient conv3 (P=3)", f"M={B * 100} N=64 K=576", us, g3.numel() * 2 + d2.numel() * 2, hbm, 2.0 * B * 100 * 64 * 576, tpk))
        wd2_all = torch.cat(wds, 1).contiguous()
        us = timeit(lambda: tc.gemm_halo(g3, wd2_all, P["h_dg2"], out_pl=d1, out_ld=32, relu_mask=act1[0]), R)
        add(entry("K12-halo data gradient conv2 (P=3, 4 phases in one launch)", f"M={B * 441} N=32 K=256", us, g3.numel() * 2 + d1.numel() * 2, hbm, 2.0 * B * 100 * 64 * 512, tpk))
        for nm, xp_, bgk, K in (("conv2", act1_pairs, "fwd2", 512), ("conv3", act2, "fwd3", 576)):
            sp = tc.wgrad_box_splits(B * P["hp2"], 6, K, 64)
            us = timeit(lambda: tc.wgrad_box(xp_, g3, P[bgk], 6, sp), R)
            add(entry("K12-box weight gradient %s (P=3, %d splits)" % (nm, sp), f"M={B * 100} N=64 K={K}", us,
                      xp_.numel() * 2 + g3.numel() * 2, hbm, 2.0 * B * 100 * 64 * K, tpk))
    if want("k13"):
        out["k13"] = k13_bench(R, hbm)
    if want("k13l"):
        out["k13l"] = k13l_bench(R)
    if want("dcg"):
        out["dcg"] = dcg_bench(R)
    print(json.dumps(out))


def k13l_bench(R, repeats=3):
    """K13L at DRQN's shapes: training (S = 8 sequences of T = 50, H = 128, input 128, configs/drqn CartPole-v1), acting
    (S = 10, T = 1) and a larger S = 640: a whole LSTM forward + backward (input projection and weight-gradient GEMMs
    included) through lstm_sequence against nn.LSTM on cuDNN (forward only for acting), both in IEEE fp32.  Each timing
    is repeated ``repeats`` times, alternating the two, so the spread is visible."""
    import subprocess
    import torch.nn as nn
    from xuance_b200.torch.rl_models import lstm_sequence
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        res = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                      "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()}
        H = I = 128
        torch.manual_seed(0)
        lstm = nn.LSTM(I, H, batch_first=True, device=DEV)
        for name, S, T, train in (("train", 8, 50, True), ("act", 10, 1, False), ("large", 640, 50, True)):
            x = torch.randn(S, T, I, device=DEV, requires_grad=train)
            dy = torch.randn(S, T, H, device=DEV)

            def step(mine):
                if not train:
                    with torch.no_grad():
                        return lstm_sequence(lstm, x)[0] if mine else lstm(x)[0]
                x.grad = None
                lstm.zero_grad(set_to_none=True)
                yy = lstm_sequence(lstm, x)[0] if mine else lstm(x)[0]
                yy.backward(dy)
            ours, cudnn = [], []
            for _ in range(repeats):
                ours.append(round(timeit(lambda: step(True), R), 2))
                cudnn.append(round(timeit(lambda: step(False), R), 2))
            res[name] = {"shape": f"S={S} T={T} H={H} I={I}" + (" fwd+bwd" if train else " fwd"), "k13l_us": ours,
                         "cudnn_us": cudnn, "speedup_median": round(float(np.median(cudnn) / np.median(ours)), 2)}
        return res
    finally:        # IEEE fp32 for this comparison only
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def k13_bench(R, hbm):
    """K13 at recurrent MAPPO's SMAC shape (S = 640 sequences of T = 60 steps, H = 64, GRU input 64): each kernel alone,
    then a whole GRU forward + backward (input projection and weight-gradient GEMMs included) through gru_sequence
    against nn.GRU on cuDNN, both in IEEE fp32, with the number of kernels each launches (torch.profiler, separate run)."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return _k13_bench(R)
    finally:        # IEEE fp32 for this comparison only
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _k13_bench(R):
    import subprocess
    import torch.nn as nn
    from xuance_b200.torch.rl_models import gru_sequence
    S, T, H, I = 640, 60, 64, 64
    res = {"shape": f"S={S} T={T} H={H} I={I}"}
    try:
        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                     "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        res["gpu"] = "nvidia-smi unavailable"
    torch.manual_seed(0)
    gru = nn.GRU(I, H, batch_first=True, device=DEV)
    x = torch.randn(S, T, I, device=DEV, requires_grad=True)
    dy = torch.randn(S, T, H, device=DEV)
    xg = torch.randn(S, T, 3 * H, device=DEV)
    w, b = gru.weight_hh_l0.detach().contiguous(), gru.bias_hh_l0.detach().contiguous()
    y, hT = torch.empty(S, T, H, device=DEV), torch.empty(S, H, device=DEV)
    gates = torch.empty(S, T, 4 * H, device=DEV)
    dxg, dgh = torch.empty(S, T, 3 * H, device=DEV), torch.empty(S, T, 3 * H, device=DEV)
    fwd = lambda: _lib.call("xb_gru_seq_fwd", _lib.ptr(xg), _lib.ptr(w), _lib.ptr(b), None, S, T, H, _lib.ptr(y),
                            _lib.ptr(hT), _lib.ptr(gates))
    bwd = lambda: _lib.call("xb_gru_seq_bwd", _lib.ptr(dy), None, _lib.ptr(w), _lib.ptr(gates), _lib.ptr(y), None, S, T,
                            H, _lib.ptr(dxg), _lib.ptr(dgh), None)
    fl = 2.0 * S * T * 3 * H * H
    res["k13_fwd_us"] = round(timeit(fwd, R), 2)
    res["k13_bwd_us"] = round(timeit(bwd, R), 2)
    res["k13_fwd_TFLOPs_fp32"] = round(fl / res["k13_fwd_us"] / 1e6, 3)

    def step(use_k13):
        x.grad = None
        gru.zero_grad(set_to_none=True)
        yy = gru_sequence(gru, x)[0] if use_k13 else gru(x)[0]
        yy.backward(dy)

    for name, k in (("gru_sequence_k13", True), ("nn_gru_cudnn", False)):
        res[name + "_fwd_bwd_us"] = round(timeit(lambda: step(k), R), 2)
        from torch.profiler import profile, ProfilerActivity
        torch.cuda.synchronize()
        try:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                step(k)
                torch.cuda.synchronize()
            res[name + "_kernels"] = sum(e.count for e in prof.key_averages() if str(e.device_type).endswith("CUDA")
                                         and not e.key.startswith(("Memcpy", "Memset")))
        except Exception as exc:     # the timing above stands without the count
            res[name + "_kernels"] = "profiler failed: %s" % exc
    return res


def dcg_bench(R):
    """K9C xb_dcg_greedy in the shape of configs/dcg/sc2/5m_vs_6m.yaml (5 agents, FULL graph: E = 10, A = 12, 8
    normalised iterations, action masks) at R = 1920 instances (one training update: 32 episodes x 60 steps) and R = 8
    (one acting step of 8 environments), against the reference's act() loop (dcg_learner.py:49-88) restated in torch on
    the same GPU (float64, scatter sums by index_add_)."""
    import subprocess
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dcg_refs
    res = {}
    try:
        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                     "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        res["gpu"] = "nvidia-smi unavailable"
    n, A, it = 5, 12, 8
    edges = dcg_refs.graph_edges(n, "FULL")
    E = len(edges)
    fr = torch.tensor([e[0] for e in edges], dtype=torch.int32, device=DEV)
    to = torch.tensor([e[1] for e in edges], dtype=torch.int32, device=DEV)
    frl, tol = fr.long(), to.long()
    for Rn in (1920, 8):
        torch.manual_seed(0)
        f = torch.randn(Rn, n, 1, A, device=DEV)
        pay = torch.randn(2, Rn, E, 1, A * A, device=DEV)
        avail = (torch.rand(Rn, n, 1, A, device=DEV) < 0.7).to(torch.uint8)
        avail[..., 0] = 1
        acts = torch.empty(Rn, n, dtype=torch.int32, device=DEV)
        k = lambda: _lib.call("xb_dcg_greedy", _lib.ptr(f), _lib.ptr(pay), pay[0].numel(), _lib.ptr(fr), _lib.ptr(to),
                              _lib.ptr(avail), A, Rn, 1, 1, 0, n, A, E, it, 1, _lib.ptr(acts), None)

        def loop():
            P = pay.reshape(2, Rn, E, A, A).clone()
            P[1] = P[1].transpose(-1, -2).clone()
            f_ij = P.mean(dim=0).double() / E
            f_ji = f_ij.transpose(-1, -2).clone()
            f_i = f.reshape(Rn, n, A).double() / n
            scat = lambda src, idx: torch.zeros(Rn, n, A, dtype=torch.float64, device=DEV).index_add_(1, idx, src)
            m_ij = torch.zeros(Rn, E, A, dtype=torch.float64, device=DEV)
            m_ji = torch.zeros(Rn, E, A, dtype=torch.float64, device=DEV)
            U = f_i + scat(m_ij, tol) + scat(m_ji, frl)
            for _ in range(it):
                jf = (U[:, frl, :] - m_ji).unsqueeze(-1) + f_ij          # both from the old messages (Jacobi)
                jb = (U[:, tol, :] - m_ij).unsqueeze(-1) + f_ji
                m_ij, m_ji = jf.max(dim=-2).values, jb.max(dim=-2).values
                m_ij = m_ij - m_ij.mean(dim=-1, keepdim=True)
                m_ji = m_ji - m_ji.mean(dim=-1, keepdim=True)
                U = f_i + scat(m_ij, tol) + scat(m_ji, frl)
            U = U.clone()
            U[avail.reshape(Rn, n, A) == 0] = -1e10
            return U.argmax(dim=-1)

        res[f"R{Rn}_xb_dcg_greedy_us"] = round(timeit(k, R, flush=False), 2)
        res[f"R{Rn}_torch_loop_us"] = round(timeit(loop, R, flush=False), 2)
        res[f"R{Rn}_speedup"] = round(res[f"R{Rn}_torch_loop_us"] / res[f"R{Rn}_xb_dcg_greedy_us"], 2)
    return res


if __name__ == "__main__":
    main()

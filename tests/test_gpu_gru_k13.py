"""GPU tests of K13 (xb_gru_seq_fwd / xb_gru_seq_bwd) and what sits on it: the kernels against the float64 restatement
over sequence counts around the 4-sequence slabs and far past one wave, T from 1 to 200, H in {1, 32, 64}, zero and
nonzero h0, with and without dhT; bit-identity from launch to launch and between S = 640 and subsets of its sequences;
the T = 1 acting step against the steps of the sequence kernel; the autograd Function against nn.GRU (cuDNN); CUDA-graph
capture; Basic_RNN_K13 against the reference's Basic_RNN fixture; and xb_rollout_store_at bit-exact."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gru_refs import gru_fwd, gru_bwd  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gru_basic_rnn.npz")
# The error relative to max(1, max|ref|), measured on an H100 over the cases below (max 3.5e-7 forward, 3.2e-7 backward)
# and stated with headroom.
TOL_FWD = 1e-6
TOL_BWD = 1e-6


def _lib():
    from xuance_b200 import _lib
    return _lib


def _problem(S, T, H, seed, nonzero_h0=True, with_dhT=True):
    """torch's default GRU initialisation scale U(+-1/sqrt(H)) and inputs of the size a LayerNorm'd MLP gives."""
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / np.sqrt(H)
    u = lambda *shape: (torch.rand(*shape, generator=g, dtype=torch.float64) * 2 - 1) * k
    p = {"xg": torch.randn(S, T, 3 * H, generator=g, dtype=torch.float64), "w_hh": u(3 * H, H), "b_hh": u(3 * H),
         "h0": torch.randn(S, H, generator=g, dtype=torch.float64) * 0.5 if nonzero_h0 else None,
         "dy": torch.randn(S, T, H, generator=g, dtype=torch.float64),
         "dhT": torch.randn(S, H, generator=g, dtype=torch.float64) if with_dhT else None}
    return {k_: None if v is None else v.float() for k_, v in p.items()}


def _dev(t):
    return None if t is None else t.to(DEV).contiguous()


def k13_fwd(xg, w_hh, b_hh, h0, gates=True):
    L = _lib()
    S, T, G = xg.shape
    H = G // 3
    y = torch.empty(S, T, H, device=DEV)
    hT = torch.empty(S, H, device=DEV)
    gt = torch.empty(S, T, 4 * H, device=DEV) if gates else None
    L.call("xb_gru_seq_fwd", L.ptr(xg), L.ptr(w_hh), L.ptr(b_hh), L.ptr(h0), S, T, H, L.ptr(y), L.ptr(hT), L.ptr(gt))
    return y, hT, gt


def k13_bwd(dy, dhT, w_hh, gates, y, h0):
    L = _lib()
    S, T, H = y.shape
    dxg = torch.empty(S, T, 3 * H, device=DEV)
    dgh = torch.empty_like(dxg)
    dh0 = torch.empty(S, H, device=DEV)
    L.call("xb_gru_seq_bwd", L.ptr(dy), L.ptr(dhT), L.ptr(w_hh), L.ptr(gates), L.ptr(y), L.ptr(h0), S, T, H,
           L.ptr(dxg), L.ptr(dgh), L.ptr(dh0))
    return dxg, dgh, dh0


def _subset(p, rows):
    """The problem restricted to the sequences `rows` (the weights are shared)."""
    r = torch.as_tensor(rows)
    return {k: v if k in ("w_hh", "b_hh") or v is None else v[r] for k, v in p.items()}


def _run(p):
    d = {k: _dev(v) for k, v in p.items()}
    y, hT, gates = k13_fwd(d["xg"], d["w_hh"], d["b_hh"], d["h0"])
    dxg, dgh, dh0 = k13_bwd(d["dy"], d["dhT"], d["w_hh"], gates, y, d["h0"])
    return {"y": y, "hT": hT, "gates": gates, "dxg": dxg, "dgh": dgh, "dh0": dh0}


def _rel_err(got, ref):
    ref = np.asarray(ref, np.float64)
    return float(np.abs(got.double().cpu().numpy() - ref).max() / max(1.0, np.abs(ref).max()))


def _check_against_float64(p, out, rows=None):
    """Compare out (or its sequences `rows`) with the float64 restatement run on the float32 inputs."""
    sel = (lambda t: t) if rows is None else (lambda t: None if t is None else t[rows])
    np_ = lambda t: None if t is None else sel(t).double().numpy()
    y, hT, gates = gru_fwd(np_(p["xg"]), p["w_hh"].double().numpy(), p["b_hh"].double().numpy(), np_(p["h0"]))
    dxg, dgh, dh0 = gru_bwd(np_(p["dy"]), np_(p["dhT"]), p["w_hh"].double().numpy(), gates, y, np_(p["h0"]))
    o = {k: (v if rows is None else v[torch.as_tensor(rows, device=DEV)]) for k, v in out.items()}
    e_f = max(_rel_err(o["y"], y), _rel_err(o["hT"], hT), _rel_err(o["gates"], gates))
    e_b = max(_rel_err(o["dxg"], dxg), _rel_err(o["dgh"], dgh), _rel_err(o["dh0"], dh0))
    print("K13 error vs float64: fwd %.3g bwd %.3g" % (e_f, e_b))
    assert e_f <= TOL_FWD and e_b <= TOL_BWD, (e_f, e_b)


CASES = [(1, 1, 1), (1, 200, 64), (31, 2, 32), (32, 60, 64), (33, 60, 1), (640, 60, 64), (640, 200, 32),
         (33, 1, 64), (5, 60, 17)]


@pytest.mark.parametrize("S,T,H", CASES)
@pytest.mark.parametrize("nonzero_h0,with_dhT", [(False, False), (True, True), (True, False), (False, True)])
def test_k13_against_float64(S, T, H, nonzero_h0, with_dhT):
    p = _problem(S, T, H, seed=S * 7 + T * 3 + H, nonzero_h0=nonzero_h0, with_dhT=with_dhT)
    _check_against_float64(p, _run(p))


def test_k13_beyond_one_wave_against_float64_and_subsets():
    S, T, H = (1 << 17) + 5, 2, 64
    p = _problem(S, T, H, seed=99)
    out = _run(p)
    rows = np.sort(np.random.default_rng(0).choice(S, 96, replace=False))
    rows[-1] = S - 1                                                   # the last, partly filled slab
    _check_against_float64(p, out, rows)
    sub = _run(_subset(p, rows))
    r = torch.as_tensor(rows, device=DEV)
    for k in out:
        assert torch.equal(out[k][r], sub[k]), k


def test_k13_bit_identical_across_launches_and_subsets():
    S, T, H = 640, 60, 64
    p = _problem(S, T, H, seed=5)
    a, b = _run(p), _run(p)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    rng = np.random.default_rng(1)
    for n in (1, 3, 37, 333):
        rows = np.sort(rng.choice(S, n, replace=False))
        sub = _run(_subset(p, rows))
        r = torch.as_tensor(rows, device=DEV)
        for k in a:
            assert torch.equal(a[k][r], sub[k]), (n, k)


def test_acting_step_is_bit_equal_to_the_sequence_kernel_steps():
    S, T, H = 24, 60, 64
    p = {k: _dev(v) for k, v in _problem(S, T, H, seed=11).items()}
    y, hT, _ = k13_fwd(p["xg"], p["w_hh"], p["b_hh"], p["h0"], gates=False)
    y_tr, _, _ = k13_fwd(p["xg"], p["w_hh"], p["b_hh"], p["h0"], gates=True)
    assert torch.equal(y, y_tr)                                        # saving the gates changes nothing
    h = p["h0"]
    for t in range(T):                                                 # T = 1 launches with the carried state
        y1, h, _ = k13_fwd(p["xg"][:, t:t + 1].contiguous(), p["w_hh"], p["b_hh"], h, gates=False)
        assert torch.equal(y1[:, 0], y[:, t]) and torch.equal(h, y[:, t]), t
    assert torch.equal(h, hT)
    zero = torch.zeros(S, H, device=DEV)
    y0, _, _ = k13_fwd(p["xg"], p["w_hh"], p["b_hh"], None, gates=False)
    y1, _, _ = k13_fwd(p["xg"][:, :1].contiguous(), p["w_hh"], p["b_hh"], zero, gates=False)
    assert torch.equal(y0[:, 0], y1[:, 0])                             # h0 = NULL is h0 = 0


def _cudnn_pair(S, T, I, H, seed):
    from xuance_b200.torch.rl_models import gru_sequence
    torch.manual_seed(seed)
    gru = nn.GRU(I, H, batch_first=True, device=DEV)
    x = torch.randn(S, T, I, device=DEV)
    h0 = torch.randn(S, H, device=DEV) * 0.5
    dy, dhT = torch.randn(S, T, H, device=DEV), torch.randn(S, H, device=DEV)
    outs = {}
    for name in ("k13", "cudnn"):
        gru.zero_grad()
        xi, hi = x.clone().requires_grad_(), h0.clone().requires_grad_()
        if name == "k13":
            y, hT = gru_sequence(gru, xi, hi)
        else:
            y, hT = gru(xi, hi[None])
            hT = hT[0]
        ((y * dy).sum() + (hT * dhT).sum()).backward()
        outs[name] = {"y": y.detach(), "hT": hT.detach(), "dx": xi.grad, "dh0": hi.grad,
                      **{n: p.grad.clone() for n, p in gru.named_parameters()}}
    return outs


@pytest.fixture
def strict_fp32():
    """cuDNN and cuBLAS in IEEE fp32 (no TF32), restored afterwards."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def test_autograd_function_against_cudnn(strict_fp32):
    for S, T, I, H in ((640, 60, 64, 64), (7, 3, 5, 1), (33, 200, 16, 32)):
        o = _cudnn_pair(S, T, I, H, seed=S + T)
        for k, c in o["cudnn"].items():
            rel = float((o["k13"][k] - c).norm() / c.norm().clamp_min(1e-30))
            print("K13 vs cuDNN", S, T, H, k, "%.3g" % rel)
            assert rel < 1e-5, (S, T, H, k, rel)


def test_autograd_function_captures_in_a_cuda_graph():
    from xuance_b200.torch.rl_models import gru_sequence
    torch.manual_seed(3)
    gru = nn.GRU(32, 64, batch_first=True, device=DEV)
    x = torch.randn(96, 60, 32, device=DEV)
    dy = torch.randn(96, 60, 64, device=DEV)

    def step():
        gru.zero_grad(set_to_none=False)
        y, _ = gru_sequence(gru, x)
        (y * dy).sum().backward()
        return y

    for p_ in gru.parameters():
        p_.grad = torch.zeros_like(p_)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            y_eager = step()
    torch.cuda.current_stream().wait_stream(side)
    g_eager = [p_.grad.clone() for p_ in gru.parameters()]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_g = step()
    for p_ in gru.parameters():
        p_.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(y_g, y_eager)
    for a, b in zip(g_eager, gru.parameters()):
        assert torch.equal(a, b.grad)


def test_basic_rnn_against_the_reference_fixture(strict_fp32):
    from xuance_b200.torch.rl_models import Basic_RNN_K13
    g = np.load(GOLDEN)
    OBS, FC, H, S, T = (int(v) for v in g["dims"])
    rep = Basic_RNN_K13((OBS,), None, normalize=nn.LayerNorm, initialize=nn.init.orthogonal_, activation=nn.ReLU,
                        device=DEV, fc_hidden_sizes=[FC], recurrent_hidden_size=H, N_recurrent_layers=1, dropout=0,
                        rnn="GRU")
    rep.load_state_dict({k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd/")}, strict=True)
    x = torch.tensor(g["x"], device=DEV, requires_grad=True)
    h0 = torch.tensor(g["h0"], device=DEV, requires_grad=True)
    o = rep(x, h0)
    (o.embeddings * torch.tensor(g["w"], device=DEV)).sum().backward()
    tol = dict(rtol=1e-4, atol=2e-5)
    np.testing.assert_allclose(o.embeddings.detach().cpu().numpy(), g["embeddings"], **tol)
    np.testing.assert_allclose(o.rnn_states.cpu().numpy(), g["hn"], **tol)
    np.testing.assert_allclose(x.grad.cpu().numpy(), g["grad/x"], **tol)
    np.testing.assert_allclose(h0.grad.cpu().numpy(), g["grad/h0"], **tol)
    for k, p_ in rep.named_parameters():
        ref = g["grad/" + k]
        np.testing.assert_allclose(p_.grad.cpu().numpy(), ref, rtol=1e-4, atol=2e-5 * max(1.0, np.abs(ref).max()),
                                   err_msg=k)
    with torch.no_grad():          # one acting step from the carried state (cuBLAS may sum the GEMMs of other M differently)
        o1 = rep(x[:, 0].detach(), h0)
    torch.testing.assert_close(o1.embeddings, o.embeddings[:, 0].detach(), rtol=1e-6, atol=1e-6)
    with torch.no_grad():
        rep.init_rnn_states_item([1, 4], o1.rnn_states)
    assert torch.count_nonzero(o1.rnn_states[:, [1, 4]]) == 0 and torch.count_nonzero(o1.rnn_states[:, 0]) > 0


def test_rollout_store_at_writes_each_row_at_its_own_step():
    L = _lib()
    N, T, F = 6, 9, 3
    rng = np.random.default_rng(4)
    for row_bytes in (48, 12):                                         # 16-byte and 4-byte paths
        W = row_bytes // 4
        dst = torch.full((N, T, W), -7.0, device=DEV)
        sdst = torch.full((F, N, T), -7.0, device=DEV)
        ref, sref = dst.cpu().numpy().copy(), sdst.cpu().numpy().copy()
        for _ in range(4):
            step = rng.integers(-1, T + 1, N).astype(np.int32)         # -1 and T: rows left alone
            src = rng.standard_normal((N, W)).astype(np.float32)
            ssrc = rng.standard_normal((F, N)).astype(np.float32)
            src_d, ssrc_d, step_d = (torch.from_numpy(a).to(DEV) for a in (src, ssrc, step))   # alive until the launch
            L.call("xb_rollout_store_at", L.ptr(dst), L.ptr(src_d), row_bytes, L.ptr(sdst), L.ptr(ssrc_d), F, N, T,
                   L.ptr(step_d))
            for n in range(N):
                if 0 <= step[n] < T:
                    ref[n, step[n]] = src[n]
                    sref[:, n, step[n]] = ssrc[:, n]
        np.testing.assert_array_equal(dst.cpu().numpy(), ref)
        np.testing.assert_array_equal(sdst.cpu().numpy(), sref)

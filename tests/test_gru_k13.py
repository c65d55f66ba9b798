"""CPU tests of K13 (the GRU sequence kernels) and the layers around it: the float64 restatement against torch.nn.GRU
autograd, the C-ABI argument checks, the no-spill ptxas check, the reference state_dict of Basic_RNN, the scope limits,
and xb_rollout_store_at's argument checks."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn as nn

from gru_refs import gru_fwd, gru_bwd, gru_param_grads

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "gru_basic_rnn.npz")
EINVAL = -1


def _torch_gru64(x, h0, p):
    gru = nn.GRU(x.shape[-1], p["w_hh"].shape[1], batch_first=True, dtype=torch.float64)
    with torch.no_grad():
        for name, v in (("weight_ih_l0", p["w_ih"]), ("weight_hh_l0", p["w_hh"]), ("bias_ih_l0", p["b_ih"]),
                        ("bias_hh_l0", p["b_hh"])):
            getattr(gru, name).copy_(torch.from_numpy(v))
    xt = torch.tensor(x, requires_grad=True)
    ht = torch.tensor(h0[None], requires_grad=True)
    y, hn = gru(xt, ht)
    return gru, xt, ht, y, hn[0]


CASES = [(1, 1, 1, 3), (1, 1, 4, 2), (3, 1, 5, 7), (2, 7, 1, 4), (4, 6, 8, 5), (2, 3, 64, 9)]   # S, T, H, I


@pytest.mark.parametrize("S,T,H,I", CASES)
@pytest.mark.parametrize("nonzero_h0", [False, True])
@pytest.mark.parametrize("with_dhT", [False, True])
def test_float64_restatement_matches_torch_gru_autograd(S, T, H, I, nonzero_h0, with_dhT):
    rng = np.random.default_rng(S * 1000 + T * 100 + H + I)
    p = {"w_ih": rng.standard_normal((3 * H, I)) * 0.6, "w_hh": rng.standard_normal((3 * H, H)) * 0.6,
         "b_ih": rng.standard_normal(3 * H) * 0.3, "b_hh": rng.standard_normal(3 * H) * 0.3}
    x = rng.standard_normal((S, T, I))
    h0 = rng.standard_normal((S, H)) if nonzero_h0 else np.zeros((S, H))
    dy = rng.standard_normal((S, T, H))
    dhT = rng.standard_normal((S, H)) if with_dhT else None
    gru, xt, ht, y, hT = _torch_gru64(x, h0, p)
    loss = (y * torch.from_numpy(dy)).sum() + ((hT * torch.from_numpy(dhT)).sum() if with_dhT else 0.0)
    loss.backward()

    xg = x @ p["w_ih"].T + p["b_ih"]
    y_r, hT_r, gates = gru_fwd(xg, p["w_hh"], p["b_hh"], h0 if nonzero_h0 else None)
    np.testing.assert_allclose(y_r, y.detach().numpy(), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(hT_r, hT.detach().numpy(), rtol=1e-12, atol=1e-13)
    dxg, dgh, dh0 = gru_bwd(dy, dhT, p["w_hh"], gates, y_r, h0 if nonzero_h0 else None)
    g = gru_param_grads(x, dxg, dgh, y_r, h0 if nonzero_h0 else None)
    np.testing.assert_allclose(dxg.reshape(-1, 3 * H) @ p["w_ih"], xt.grad.numpy().reshape(-1, I), rtol=1e-11,
                               atol=1e-12)
    np.testing.assert_allclose(dh0, ht.grad.numpy()[0], rtol=1e-11, atol=1e-12)
    for name, key in (("weight_ih_l0", "dW_ih"), ("weight_hh_l0", "dW_hh"), ("bias_ih_l0", "db_ih"),
                      ("bias_hh_l0", "db_hh")):
        np.testing.assert_allclose(g[key], getattr(gru, name).grad.numpy(), rtol=1e-11, atol=1e-12, err_msg=name)


def test_gru_entry_points_validate_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    j = ctypes.c_void_p(0x1000)
    for name in ("xb_gru_seq_fwd", "xb_gru_seq_bwd", "xb_rollout_store_at"):
        assert name in _lib.exported_symbols() and hasattr(lib, name)

    def fwd(S=8, T=4, H=16, xg=j, w=j, b=j, h0=None, y=j, hT=j, gates=None):
        return lib.xb_gru_seq_fwd(xg, w, b, h0, S, T, H, y, hT, gates, None)

    def bwd(S=8, T=4, H=16, dy=j, dhT=None, w=j, gates=j, y=j, h0=None, dxg=j, dgh=j, dh0=None):
        return lib.xb_gru_seq_bwd(dy, dhT, w, gates, y, h0, S, T, H, dxg, dgh, dh0, None)
    for f in (fwd, bwd):
        assert f(S=0) == EINVAL and f(S=-3) == EINVAL
        assert f(T=0) == EINVAL and f(T=-1) == EINVAL
        assert f(H=0) == EINVAL and f(H=65) == EINVAL and f(H=-1) == EINVAL     # outside 1..64
    for k in ("xg", "w", "b", "y", "hT"):
        assert fwd(**{k: None}) == EINVAL, k
    for k in ("dy", "w", "gates", "y", "dxg", "dgh"):
        assert bwd(**{k: None}) == EINVAL, k

    def store_at(N=4, T=8, F=2, step=j, rd=j, rs=j, sd=j, ss=j, rb=16):
        return lib.xb_rollout_store_at(rd, rs, rb, sd, ss, F, N, T, step, None)
    assert store_at(step=None) == EINVAL and store_at(N=0) == EINVAL and store_at(T=0) == EINVAL
    assert store_at(F=-1) == EINVAL and store_at(rd=None) == EINVAL and store_at(sd=None) == EINVAL
    assert store_at(rb=6) == -2                                                     # XB_EALIGN: row_bytes % 4 != 0


@pytest.mark.skipif(not (shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc")), reason="nvcc not available")
def test_gru_kernels_do_not_spill(tmp_path):
    from xuance_b200 import build
    flags = [f for f in build.NVCC_FLAGS if f not in ("--use_fast_math=false", "-shared")]
    cmd = [build._nvcc()] + flags + ["-c", os.path.join(build.CSRC, "gru.cu"), "-o", str(tmp_path / "gru.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S*gru_seq_\S*)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = sum(int(v) for v in m.groups())
            cur = None
    assert len(kernels) == 2, log
    assert kernels == {k: 0 for k in kernels}, log


def _rep(device="cpu", **kw):
    from xuance_b200.torch.rl_models import Basic_RNN_K13
    args = dict(fc_hidden_sizes=[64], recurrent_hidden_size=64, N_recurrent_layers=1, dropout=0, rnn="GRU")
    args.update(kw)
    return Basic_RNN_K13((30,), None, normalize=nn.LayerNorm, initialize=nn.init.orthogonal_, activation=nn.ReLU,
                         device=device, **args)


def test_basic_rnn_loads_the_reference_state_dict_strictly_and_keeps_its_initialisation():
    g = np.load(GOLDEN)
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd/")}
    rep = _rep()
    assert set(rep.state_dict()) == set(sd)
    for k, v in rep.state_dict().items():
        assert tuple(v.shape) == tuple(sd[k].shape), k
    rep.load_state_dict(sd, strict=True)
    fresh = _rep()
    for k, v in fresh.state_dict().items():                     # gru_block / mlp_block: orthogonal weights, zero biases
        if k.endswith("bias") and not k.startswith(("input_norm", "norm_rnn")) and "mlp.2" not in k:
            assert torch.count_nonzero(v) == 0, k
    w = fresh.rnn.weight_hh_l0.detach()
    torch.testing.assert_close(w.T @ w, torch.eye(64), atol=1e-5, rtol=0)


def test_scope_limits_raise_named_errors():
    with pytest.raises(NotImplementedError, match="LSTM"):
        _rep(rnn="LSTM")
    with pytest.raises(NotImplementedError, match="N_recurrent_layers"):
        _rep(N_recurrent_layers=2)
    with pytest.raises(NotImplementedError, match="dropout"):
        _rep(dropout=0.1)
    with pytest.raises(NotImplementedError, match="1..64"):
        _rep(recurrent_hidden_size=65)
    from xuance_b200.torch.rl_models import GRUSequence
    with pytest.raises(NotImplementedError, match="1..64"):
        GRUSequence.apply(torch.zeros(2, 3, 3 * 96), torch.zeros(3 * 96, 96), torch.zeros(3 * 96), None)


def test_qmix_keeps_its_cudnn_gru():
    from xuance_b200.torch.rl_models import Basic_RNN
    from xuance_b200.torch.rl_models.representations import REGISTRY_Representation
    assert REGISTRY_Representation["Basic_RNN"] is Basic_RNN
    rep = Basic_RNN((30,), fc_hidden_sizes=[64], recurrent_hidden_size=64, activation=nn.ReLU, device="cpu")
    assert isinstance(rep.rnn, nn.GRU) and type(rep).forward is not type(_rep()).forward

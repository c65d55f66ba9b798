"""CPU tests of DRQN: the float64 LSTM restatement against torch.nn.LSTM autograd, the torch-CPU oracle against the
reference fixture, the strict load of the reference's state_dict, K13L's C-ABI argument checks and its no-spill ptxas
report, and the config, registries and scope errors."""
import ctypes
import os
import re
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn as nn

from lstm_refs import lstm_fwd, lstm_bwd, lstm_param_grads
from oracle_drqn import DRQNOracle, DRQNLearnerOracle, seeded_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "drqn_update.npz")
EINVAL = -1
# name, rnn, H, obs_dim, rep hidden, n_actions, B, lookup, windows, grad clip, seed (tests/golden/make_golden_drqn.py)
CASES = [("lstm128", "LSTM", 128, 4, 16, 2, 8, 50, (50, 50, 20, 20), False, 11),
         ("lstm17", "LSTM", 17, 5, 24, 3, 5, 12, (12, 7, 7, 12), True, 12),
         ("gru64", "GRU", 64, 4, 32, 2, 6, 10, (10, 6, 6, 10), True, 13)]
FULL_CASE = "lstm17"      # recorded in full from the reference's own initialisation; the others start from seeded_state


@pytest.mark.parametrize("S,T,H,I", [(1, 1, 1, 3), (1, 1, 17, 4), (1, 1, 128, 5), (3, 6, 17, 4), (2, 4, 128, 3)])
@pytest.mark.parametrize("nonzero_state", [False, True])
@pytest.mark.parametrize("with_dT", [False, True])
def test_float64_restatement_matches_torch_lstm_autograd(S, T, H, I, nonzero_state, with_dT):
    rng = np.random.default_rng(S * 1000 + T * 100 + H + I)
    p = {"w_ih": rng.standard_normal((4 * H, I)) * 0.5, "w_hh": rng.standard_normal((4 * H, H)) * (0.5 / np.sqrt(H)),
         "b_ih": rng.standard_normal(4 * H) * 0.3, "b_hh": rng.standard_normal(4 * H) * 0.3}
    x = rng.standard_normal((S, T, I))
    h0 = rng.standard_normal((S, H)) if nonzero_state else np.zeros((S, H))
    c0 = rng.standard_normal((S, H)) if nonzero_state else np.zeros((S, H))
    dy = rng.standard_normal((S, T, H))
    dhT = rng.standard_normal((S, H)) if with_dT else None
    dcT = rng.standard_normal((S, H)) if with_dT else None
    lstm = nn.LSTM(I, H, batch_first=True, dtype=torch.float64)
    with torch.no_grad():
        for name, key in (("weight_ih_l0", "w_ih"), ("weight_hh_l0", "w_hh"), ("bias_ih_l0", "b_ih"),
                          ("bias_hh_l0", "b_hh")):
            getattr(lstm, name).copy_(torch.from_numpy(p[key]))
    xt = torch.tensor(x, requires_grad=True)
    ht, ct = torch.tensor(h0[None], requires_grad=True), torch.tensor(c0[None], requires_grad=True)
    y, (hT, cT) = lstm(xt, (ht, ct))
    loss = (y * torch.from_numpy(dy)).sum()
    if with_dT:
        loss = loss + (hT[0] * torch.from_numpy(dhT)).sum() + (cT[0] * torch.from_numpy(dcT)).sum()
    loss.backward()

    xg = x @ p["w_ih"].T + p["b_ih"]
    s0 = (h0, c0) if nonzero_state else (None, None)
    y_r, hT_r, cT_r, gates = lstm_fwd(xg, p["w_hh"], p["b_hh"], *s0)
    np.testing.assert_allclose(y_r, y.detach().numpy(), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(hT_r, hT[0].detach().numpy(), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(cT_r, cT[0].detach().numpy(), rtol=1e-12, atol=1e-13)
    dxg, dh0, dc0 = lstm_bwd(dy, dhT, dcT, p["w_hh"], gates, s0[1])
    np.testing.assert_allclose(dxg.reshape(-1, 4 * H) @ p["w_ih"], xt.grad.numpy().reshape(-1, I), rtol=1e-11,
                               atol=1e-12)
    np.testing.assert_allclose(dh0, ht.grad.numpy()[0], rtol=1e-11, atol=1e-12)
    np.testing.assert_allclose(dc0, ct.grad.numpy()[0], rtol=1e-11, atol=1e-12)
    g = lstm_param_grads(x, dxg, y_r, s0[0])
    for name, key in (("weight_ih_l0", "dW_ih"), ("weight_hh_l0", "dW_hh"), ("bias_ih_l0", "db_ih"),
                      ("bias_hh_l0", "db_hh")):
        np.testing.assert_allclose(g[key], getattr(lstm, name).grad.numpy(), rtol=1e-11, atol=1e-12, err_msg=name)


def _golden():
    return np.load(GOLDEN)


def _state(z, prefix):
    return {k[len(prefix):]: torch.from_numpy(z[k].copy()) for k in z.files if k.startswith(prefix)}


def _digest(v):
    v = np.asarray(v, np.float64)
    return np.array([v.sum(), np.abs(v).sum()])


def initial_state(z, case, template):
    """The case's initial weights: the reference's (recorded) for FULL_CASE, seeded_state over ``template`` otherwise."""
    if case[0] == FULL_CASE:
        return _state(z, f"{case[0]}/init/")
    return seeded_state(template, case[10])


def as_recorded(name, v):
    return v if name == FULL_CASE else _digest(v)


def run_oracle(z, case):
    name, rnn, H, obs_dim, rep_hidden, A, B, lookup, windows, clip, seed = case
    model = DRQNOracle(rnn, H, obs_dim, rep_hidden, A)
    model.load_state_dict(initial_state(z, case, model.state_dict()), strict=True)
    learner = DRQNLearnerOracle(model, use_grad_clip=clip)
    infos = []
    for u in range(len(windows)):
        s = {k: z[f"{name}/u{u}/{k}"] for k in ("obs", "actions", "rewards", "terminals")}
        infos.append(learner.update(**s))
    return model, learner, infos


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_reproduces_reference_fixture(case):
    z = _golden()
    name = case[0]
    model, learner, infos = run_oracle(z, case)
    for u, info in enumerate(infos):
        for k in ("Qloss", "learning_rate", "predictQ"):
            np.testing.assert_allclose(info[k], float(z[f"{name}/u{u}/info/{k}"]), rtol=1e-5, atol=1e-7,
                                       err_msg=f"{name} u{u} {k}")
    for k, v in model.state_dict().items():
        ref = z[f"{name}/final/{k}"]
        got = as_recorded(name, v.numpy())
        np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-6, err_msg=k)
    pnames = dict(model.named_parameters())
    for pname, p in pnames.items():
        st = learner.optimizer.state.get(p)
        if not st:
            continue
        for m in ("exp_avg", "exp_avg_sq"):
            got = as_recorded(name, st[m].numpy())
            np.testing.assert_allclose(got, z[f"{name}/adam/{m}/{pname}"], rtol=1e-4, atol=1e-9,
                                       err_msg=f"{pname} {m}")


def _config(rnn="LSTM", H=128, **kw):
    cfg = dict(representation="Basic_MLP", representation_hidden_size=[16], recurrent_hidden_size=H,
               recurrent_layer_N=1, dropout=0, rnn=rnn, activation="relu")
    cfg.update(kw)
    return SimpleNamespace(**cfg)


def _model(rnn="LSTM", H=128, obs_dim=4, rep_hidden=16, A=2, layers=1, dropout=0, action_space=None):
    from xuance_b200.common import Discrete
    from xuance_b200.torch.rl_models import Basic_MLP, DeepRecurrentQNetwork
    rep = Basic_MLP((obs_dim,), [rep_hidden], None, nn.init.orthogonal_, nn.ReLU, None)
    return DeepRecurrentQNetwork(rep, H, layers, dropout, action_space or Discrete(A), rnn, nn.init.orthogonal_, None)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_reference_state_dict_loads_strict(case):
    """Every case's recorded final state_dict names are the network's; FULL_CASE's reference initialisation loads with
    strict=True and equals the one this package builds from the same torch seed."""
    z = _golden()
    name, rnn, H, obs_dim, rep_hidden, A = case[:6]
    seed = case[10]
    torch.manual_seed(seed)
    model = _model(rnn, H, obs_dim, rep_hidden, A)
    prefix = f"{name}/final/"
    assert list(model.state_dict()) == [k[len(prefix):] for k in z.files if k.startswith(prefix)]   # seeded_state order
    if name == FULL_CASE:
        sd = _state(z, f"{name}/init/")
        for k, v in model.state_dict().items():
            assert torch.equal(v, sd[k]), k
        model.load_state_dict(sd, strict=True)
    else:
        model.load_state_dict(seeded_state(model.state_dict(), seed), strict=True)


def test_scope_errors():
    from xuance_b200.common import Box
    with pytest.raises(NotImplementedError, match="1..128"):
        _model("LSTM", 129)
    with pytest.raises(NotImplementedError, match="1..128"):
        _model("LSTM", 512)                      # the Atari and CarRacing configs
    with pytest.raises(NotImplementedError, match="1..64"):
        _model("GRU", 65)
    with pytest.raises(NotImplementedError, match="recurrent_layer_N"):
        _model("LSTM", 64, layers=2)
    with pytest.raises(NotImplementedError, match="dropout"):
        _model("LSTM", 64, dropout=0.1)
    with pytest.raises(ValueError, match="Discrete"):
        _model("LSTM", 64, action_space=Box(-1.0, 1.0, (2,)))
    with pytest.raises(ValueError, match="Unknown recurrent"):
        _model("RNN", 64)


def test_config_and_registries():
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents, DRQN_Agent
    from xuance_b200.torch.learners import REGISTRY_Learners, DRQN_Learner
    # DRQN_Agent builds its learner through REGISTRY_Learners[config.learner]; the agent itself is constructed directly
    assert REGISTRY_Learners["DRQN_Learner"] is DRQN_Learner
    assert DRQN_Agent not in REGISTRY_Agents.values()
    cfg = get_arguments("drqn", "classic_control", "CartPole-v1")
    assert (cfg.agent, cfg.learner, cfg.rnn, cfg.recurrent_hidden_size, cfg.lookup_length) == \
        ("DRQN", "DRQN_Learner", "LSTM", 128, 50)
    for env_id, env in (("Acrobot-v1", "classic_control"), ("MountainCar-v0", "classic_control"),
                        ("LunarLander-v3", "box2d"), ("CarRacing-v3", "box2d"), ("Breakout-v5", "atari")):
        with pytest.raises(AttributeError, match="no config"):
            get_arguments("drqn", env, env_id)


def test_drqn_config_defines_every_key_its_classes_read():
    """The static check of test_host_logic.py's shipped-config test, for configs/drqn/classic_control/CartPole-v1.yaml
    (that test reads configs/<algo>/*.yaml only): every ``config.X`` DRQN_Agent, DRQN_Learner and their bases read
    without a getattr / hasattr default is a key of basic.yaml or of the DRQN yaml."""
    import yaml
    root = os.path.join(ROOT, "xuance_b200")
    rd = lambda *p: open(os.path.join(root, *p)).read()
    base = set(yaml.safe_load(rd("configs", "basic.yaml")))
    cfg = yaml.safe_load(rd("configs", "drqn", "classic_control", "CartPole-v1.yaml"))
    files = ["torch/agents/agent.py", "torch/agents/off_policy.py", "torch/agents/drqn_agent.py",
             "torch/learners/learner.py", "torch/learners/dqn_learner.py", "torch/learners/drqn_learner.py"]
    src = "".join(rd(*f.split("/")) for f in files)
    hard = set(re.findall(r"(?<![a-zA-Z_])(?:self\.)?config\.([a-zA-Z_][a-zA-Z0-9_]*)\b(?!\s*=[^=])", src))
    soft = set(re.findall(r"(?:getattr|hasattr)\((?:self\.)?config,\s*.([a-zA-Z_0-9]+).", src))
    assert {"rnn", "lookup_length", "recurrent_hidden_size", "decay_step_greedy"} <= hard
    assert not sorted(hard - soft - base - set(cfg))


def test_lstm_entry_points_validate_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    j = ctypes.c_void_p(0x1000)
    for name in ("xb_lstm_seq_fwd", "xb_lstm_seq_bwd"):
        assert name in _lib.exported_symbols() and hasattr(lib, name)

    def fwd(S=8, T=4, H=16, xg=j, w=j, b=j, h0=None, c0=None, y=j, hT=j, cT=j, gates=None):
        return lib.xb_lstm_seq_fwd(xg, w, b, h0, c0, ctypes.c_int64(S), T, H, y, hT, cT, gates, None)

    def bwd(S=8, T=4, H=16, dy=j, dhT=None, dcT=None, w=j, gates=j, c0=None, dxg=j, dh0=None, dc0=None):
        return lib.xb_lstm_seq_bwd(dy, dhT, dcT, w, gates, c0, ctypes.c_int64(S), T, H, dxg, dh0, dc0, None)
    for f in (fwd, bwd):
        assert f(S=0) == EINVAL and f(S=-3) == EINVAL
        assert f(S=(1 << 33)) == EINVAL                 # more slabs than a grid holds
        assert f(T=0) == EINVAL and f(T=-1) == EINVAL
        assert f(H=0) == EINVAL and f(H=129) == EINVAL and f(H=-1) == EINVAL
    for kw in ("xg", "w", "b", "y", "hT", "cT"):
        assert fwd(**{kw: None}) == EINVAL, kw
    for kw in ("dy", "w", "gates", "dxg"):
        assert bwd(**{kw: None}) == EINVAL, kw


def test_lstm_entry_points_raise_from_python():
    from xuance_b200.torch.rl_models.lstm import LSTMSequence
    with pytest.raises(NotImplementedError, match="1..128"):
        LSTMSequence.apply(torch.zeros(1, 1, 4 * 129), torch.zeros(4 * 129, 129), torch.zeros(4 * 129), None, None)


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"),
                    reason="nvcc not available")
def test_k13l_kernels_do_not_spill(tmp_path):
    from xuance_b200 import build
    flags = [f for f in build.NVCC_FLAGS if f not in ("--use_fast_math=false", "-shared")]
    res = subprocess.run([build._nvcc()] + flags + ["-c", os.path.join(build.CSRC, "lstm.cu"), "-o",
                                                    str(tmp_path / "lstm.o")], capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    found, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S*lstm_seq_(fwd|bwd)_kernel\S*)'", line)
        if m:
            cur = m.group(2)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            found[cur] = int(m.group(1)) + int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if cur and m:
            assert int(m.group(1)) * 512 <= 65536, line     # 4H = 512 threads at H = 128 must fit one SM's registers
            cur = None
    assert found == {"fwd": 0, "bwd": 0}, log

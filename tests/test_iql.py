"""CPU tests of IQL: the float64 restatement of K9I (tests/iql_refs.py) against float64 autograd of the reference's
expressions and hand-computed cases (ties, an all-unavailable next row, d = 1, A = 1 and n = 1, M = 0), the K9I argument
checks, ptxas on iql.cu, the shipped configs, the registries, the out-of-scope errors and the epsilon schedule; the
torch-CPU oracle (tests/oracle_iql.py) against every update of the reference fixture."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import iql_refs as R
from xuance_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _one(q_all, q_tgt, actions, rewards, terminals, mask=None, filled=None, avail=None):
    B, n, T1, _ = q_all.shape
    T = T1 - 1
    mask = torch.ones(B, n, T, dtype=q_all.dtype) if mask is None else mask
    filled = torch.ones(B, T, dtype=q_all.dtype) if filled is None else filled
    return (q_all, q_tgt, actions, rewards, terminals, mask, filled, avail)


# ---------------------------------------------------------------- the restatement
@pytest.mark.parametrize("double_q", [True, False])
@pytest.mark.parametrize("masked", [True, False])
@pytest.mark.parametrize("B,n,T,A", [(1, 1, 1, 1), (2, 3, 5, 4), (3, 1, 7, 9), (2, 5, 4, 12)])
def test_closed_form_gradient_matches_float64_autograd(double_q, masked, B, n, T, A):
    rng = np.random.default_rng(B * 1000 + n * 100 + T * 10 + A)
    x = R.inputs(rng, B, n, T, A, masked=masked, dtype=np.float64)
    q_all = x["q_all"].clone().requires_grad_(True)
    args = (q_all, x["q_tgt"], x["actions"], x["rewards"], x["terminals"], x["agent_mask"], x["filled"], x["avail"],
            double_q, 0.99)
    loss, pq = R.forward(*args)[:2]
    loss.backward()
    stats, dq = R.grads(x["q_all"], *args[1:])
    torch.testing.assert_close(stats, torch.stack([loss.detach(), pq.detach()]), rtol=1e-12, atol=0)
    torch.testing.assert_close(dq, q_all.grad, rtol=1e-12, atol=1e-15)
    assert not dq[:, :, -1].any()                                       # step T carries no gradient


def test_ties_take_the_first_index_and_an_all_unavailable_row_targets_minus_1e10():
    q_all = torch.tensor([[[[0.0, 0.0, 0.0], [2.0, 5.0, 5.0]]]], dtype=torch.float64)     # [1, 1, T+1=2, 3]
    q_tgt = torch.tensor([[[[0.0, 0.0, 0.0], [1.0, 3.0, 7.0]]]], dtype=torch.float64)
    a, r, d = torch.zeros(1, 1, 1, dtype=torch.float64), torch.ones(1, 1, 1, dtype=torch.float64), torch.zeros(1, 1, 1)
    _, _, nxt, qn, y, _ = R.forward(*_one(q_all, q_tgt, a, r, d.double()), True, 0.5)
    assert nxt.tolist() == [[[1]]] and qn.tolist() == [3.0] and y.tolist() == [2.5]      # tie 5 / 5: index 1
    _, _, nxt, qn, _, _ = R.forward(*_one(q_all, q_tgt, a, r, d.double()), False, 0.5)
    assert qn.tolist() == [7.0]                                                          # max of the target row
    av = torch.tensor([[[[1, 1, 1], [0, 0, 0]]]], dtype=torch.uint8)
    for double_q in (True, False):
        _, _, nxt, qn, y, _ = R.forward(*_one(q_all, q_tgt, a, r, d.double(), avail=av), double_q, 0.5)
        assert nxt.tolist() == [[[0]]] and qn.tolist() == [-1e10] and y.tolist() == [1.0 - 0.5e10]


def test_terminal_steps_drop_the_bootstrap_and_dead_or_padded_rows_drop_out():
    q_all = torch.zeros(1, 2, 3, 2, dtype=torch.float64)
    q_all[0, 0, 0, 1] = 4.0
    q_tgt = torch.full((1, 2, 3, 2), 9.0, dtype=torch.float64)
    actions = torch.tensor([[[1.0, 0.0], [0.0, 0.0]]], dtype=torch.float64)
    rewards = torch.tensor([[[1.0, 2.0], [3.0, 4.0]]], dtype=torch.float64)
    terminals = torch.tensor([[[1.0, 0.0], [0.0, 0.0]]], dtype=torch.float64)
    mask = torch.tensor([[[1.0, 1.0], [0.0, 1.0]]], dtype=torch.float64)                 # agent 1 dead at step 0
    filled = torch.tensor([[1.0, 0.0]], dtype=torch.float64)                             # step 1 padded
    stats, dq = R.grads(*_one(q_all, q_tgt, actions, rewards, terminals, mask, filled), True, 0.5)
    td = 4.0 - 1.0                                                                       # d = 1: y = r
    assert stats.tolist() == [td ** 2 / 1.0, 4.0 / 4]
    want = torch.zeros_like(q_all)
    want[0, 0, 0, 1] = 2 * td
    assert torch.equal(dq, want)


def test_a1_n1_and_the_empty_mask():
    q_all = torch.tensor([[[[1.5], [2.0]]]], dtype=torch.float64)
    q_tgt = torch.tensor([[[[0.0], [4.0]]]], dtype=torch.float64)
    a = torch.zeros(1, 1, 1, dtype=torch.float64)
    r, d = torch.ones(1, 1, 1, dtype=torch.float64), torch.zeros(1, 1, 1, dtype=torch.float64)
    stats, dq = R.grads(*_one(q_all, q_tgt, a, r, d), False, 0.5)
    assert stats.tolist() == [(1.5 - 3.0) ** 2, 1.5] and dq[0, 0, 0, 0].item() == 2 * (1.5 - 3.0)
    stats, dq = R.grads(*_one(q_all, q_tgt, a, r, d, mask=torch.zeros(1, 1, 1, dtype=torch.float64)), False, 0.5)
    assert np.isnan(stats[0].item()) and stats[1].item() == 1.5                          # 0/0, as the reference
    assert np.isnan(dq[0, 0, 0, 0].item())


# ---------------------------------------------------------------- ABI, ptxas
def test_abi_symbols_and_argument_checks_without_gpu():
    from xuance_b200 import _lib
    for s in ("xb_iql_prepare", "xb_iql_td_fwd_bwd"):
        assert s in _lib.exported_symbols()
    lib = _lib.load()
    EINVAL, ERANGE = -1, -3
    j = 256  # any non-NULL pointer: validation returns before the device is touched
    prep = lambda **k: lib.xb_iql_prepare(k.get("m", j), j, k.get("B", 4), 5, 6, k.get("out", j), j, None)
    assert prep(B=0) == EINVAL and prep(m=None) == EINVAL and prep(out=None) == EINVAL
    td = lambda **k: lib.xb_iql_td_fwd_bwd(j, k.get("qt", j), *([j] * 5), k.get("av"), k.get("ld", 0), j,
                                           k.get("B", 4), k.get("n", 5), 6, k.get("A", 12), 1, 0.99,
                                           k.get("rows", 120), j, j, j, None, None, None, None)
    assert td(qt=None) == EINVAL and td(B=0) == EINVAL and td(rows=119) == EINVAL
    assert td(av=j, ld=11) == EINVAL and td(n=33, rows=10**6) == ERANGE and td(A=65) == ERANGE


def test_iql_kernels_compile_without_spills(tmp_path):
    flags = [f for f in build.NVCC_FLAGS if f not in ("--use_fast_math=false", "-shared")]
    cmd = [build._nvcc()] + flags + ["-c", os.path.join(build.CSRC, "iql.cu"), "-o", str(tmp_path / "iql.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S*iql\S*)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = sum(int(x) for x in m.groups())
            cur = None
    assert len(kernels) == 2, log
    assert {k: v for k, v in kernels.items() if v} == {}


# ---------------------------------------------------------------- configs, registries, scope, epsilon
def test_shipped_configs_define_every_key_their_classes_read():
    import yaml
    from xuance_b200.common.common_tools import get_arguments
    pkg = os.path.join(ROOT, "xuance_b200")
    rd = lambda *p: open(os.path.join(pkg, *p)).read()
    marl = rd("torch", "agents", "marl.py")
    marl = marl[:marl.index("class QMIX_Agents")]                      # IQL_Agents' bases only
    src = marl + "".join(rd(*f.split("/")) for f in ("torch/agents/iql_agents.py", "torch/learners/iql_learner.py",
                                                      "torch/learners/qmix_learner.py", "torch/agents/agent.py",
                                                      "torch/learners/learner.py"))
    hard = set(re.findall(r"(?<![a-zA-Z_])(?:self\.)?config\.([a-zA-Z_][a-zA-Z0-9_]*)\b(?!\s*=[^=])", src))
    hard |= set(re.findall(r"(?<![a-zA-Z_])(?:c|cfg)\.([a-zA-Z_][a-zA-Z0-9_]*)\b(?!\s*=[^=])", rd("torch", "agents",
                                                                                                 "iql_agents.py")))
    soft = set(re.findall(r"(?:getattr|hasattr)\((?:self\.)?(?:config|c|cfg),\s*.([a-zA-Z_0-9]+).", src))
    base = set(yaml.safe_load(rd("configs", "basic.yaml")))
    for env_id in ("3m", "5m_vs_6m"):
        raw = yaml.safe_load(rd("configs", "iql", "sc2", f"{env_id}.yaml"))
        assert not sorted(hard - soft - base - set(raw)), (env_id, sorted(hard - soft - base - set(raw)))
        cfg = get_arguments("iql", "sc2", env_id)
        assert cfg.env_id == env_id and cfg.agent == "IQL" and cfg.learner == "IQL_Learner"
        assert cfg.use_rnn and cfg.rnn == "GRU" and cfg.use_actions_mask and cfg.double_q
        assert cfg.recurrent_hidden_size == 64 and cfg.q_hidden_size == [64] and cfg.sync_frequency == 200


def test_registries():
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    assert REGISTRY_Agents["IQL"].__name__ == "IQL_Agents"
    assert REGISTRY_Learners["IQL_Learner"].__name__ == "IQL_Learner"
    assert REGISTRY_Agents["QMIX"].__name__ == "QMIX_Agents" and REGISTRY_Learners["QMIX_Learner"].__name__ == "QMIX_Learner"


def _cfg(**over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("iql", "sc2", "3m")
    cfg.device = "cpu"
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def _spaces(n=3, A=6, box=False):
    from xuance_b200.common import Box, Discrete
    keys = [f"a{i}" for i in range(n)]
    act = {k: Box(-1, 1, (2,)) if box else Discrete(A) for k in keys}
    return dict(num_agents=n, agent_keys=keys, state_space=Box(-1, 1, (10,)),
                observation_space={k: Box(-1, 1, (8,)) for k in keys}, action_space=act)


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import IQL_Learner
    IQL = REGISTRY_Agents["IQL"]
    for over, match in ((dict(use_rnn=False), "use_rnn"), (dict(rnn="LSTM"), "LSTM"),
                        (dict(N_recurrent_layers=2), "N_recurrent_layers"),
                        (dict(recurrent_hidden_size=65), "recurrent_hidden_size"),
                        (dict(use_parameter_sharing=False), "parameter-sharing"),
                        (dict(qmix_rnn_detach_q_eval=True), "nothing would train")):
        with pytest.raises(NotImplementedError, match=match):
            IQL(_cfg(**over), **_spaces())
    with pytest.raises(NotImplementedError, match="64 actions"):
        IQL(_cfg(), **_spaces(A=65))
    with pytest.raises(NotImplementedError, match="32 agents"):
        IQL(_cfg(), **_spaces(n=33))
    with pytest.raises(ValueError, match="Discrete"):
        IQL(_cfg(), **_spaces(box=True))
    with pytest.raises(NotImplementedError, match="use_rnn"):
        IQL_Learner(_cfg(use_rnn=False), None, None, None)
    with pytest.raises(NotImplementedError, match="nothing would train"):
        IQL_Learner(_cfg(qmix_rnn_detach_q_eval=True), None, None, None)


def test_epsilon_decays_per_environment_step(monkeypatch):
    """iql_agents.py:36-38: delta = (start - end) / decay_step_greedy, applied to the environment step count (QMIX divides
    decay_step_greedy by the number of envs)."""
    from xuance_b200.torch.agents import REGISTRY_Agents
    IQL = REGISTRY_Agents["IQL"]
    for name in ("_build_model", "_build_memory", "_build_learner"):
        monkeypatch.setattr(IQL, name, lambda self, *a: None)
    ag = IQL(_cfg(start_greedy=1.0, end_greedy=0.05, decay_step_greedy=50000, parallels=8), **_spaces())
    assert ag.e_greedy == 1.0 and ag.delta_egreedy == pytest.approx(0.95 / 50000)
    ag.current_step = 10000
    ag._update_explore_factor()
    assert ag.e_greedy == pytest.approx(1.0 - 0.95 * 10000 / 50000)
    ag.current_step = 60000
    ag._update_explore_factor()
    assert ag.e_greedy < 0.05
    ag._update_explore_factor()
    assert ag.e_greedy == 0.05


def test_independent_mixer_passes_values_through():
    from xuance_b200.torch.rl_models import IndependentMixer
    m = IndependentMixer()
    x = torch.randn(4, 3)
    assert m(x, None) is x and not list(m.parameters())


# ---------------------------------------------------------------- the reference fixture (tests/golden/iql_update.npz)
GOLDEN = os.path.join(ROOT, "tests", "golden", "iql_update.npz")
# as make_golden_iql.py records them
FIX_OBS, FIX_A, FIX_T, FIX_HID = 12, 7, 8, 16
FIX_UPDATES = 4
FIX_CASES = [(n, dq, mask) for n in (1, 3) for dq in (True, False) for mask in (True, False)]
FIX_INFO_KEYS = ("loss_Q", "predictQ", "learning_rate")


def case_name(n, double_q, mask):
    return f"n{n}/dq{int(double_q)}/m{int(mask)}/"


def fixture_init(d, pre):
    return {k[len(pre) + 5:]: torch.from_numpy(d[k]) for k in d.files if k.startswith(pre + "init/")}


def fixture_sample(d, pre, it, keys):
    p = f"{pre}in{it}/"
    s = {f: {k: d[p + f][:, i] for i, k in enumerate(keys)}
         for f in ("obs", "actions", "rewards", "terminals", "agent_mask", "avail_actions")}
    B, T = d[p + "filled"].shape
    s.update(filled=d[p + "filled"], batch_size=B, sequence_length=T)
    return s


def test_reference_state_dict_loads_strictly_and_the_unmodified_reference_does_not_train():
    """The unmodified reference raises on the agent-axis slice of the masks; without masks it runs, but its q_eval was
    sliced under no_grad and no parameter moves."""
    from oracle_iql import build_model
    d = np.load(GOLDEN)
    for n, dq, mask in FIX_CASES:
        pre = case_name(n, dq, mask)
        _, _, model = build_model(n, FIX_OBS, FIX_A, FIX_HID, "cpu")
        model.load_state_dict(fixture_init(d, pre), strict=True)
        what = str(d[pre + "unmodified"])
        if mask:
            assert what.startswith("IndexError: The shape of the mask"), what
        else:
            assert what == "ran: parameters unchanged", what


@pytest.mark.parametrize("n,double_q,mask", FIX_CASES)
def test_oracle_reproduces_the_reference_fixture(n, double_q, mask):
    """The float64 oracle against every update of the reference (float32): the greedy next actions exactly, the logged
    values within 1e-5 relative, the whole state_dict after every update within 1e-5 + 1e-5 relative."""
    from oracle_iql import IQLOracle, build_model
    d = np.load(GOLDEN)
    pre = case_name(n, double_q, mask)
    keys, _, model = build_model(n, FIX_OBS, FIX_A, FIX_HID, "cpu")
    model.load_state_dict(fixture_init(d, pre), strict=True)
    orc = IQLOracle(model, double_q=double_q, total_iters=int(d[pre + "total_iters"]), use_actions_mask=mask)
    for it in range(FIX_UPDATES):
        s = fixture_sample(d, pre, it, keys)
        nxt = orc.forward(s)[2]
        np.testing.assert_array_equal(nxt.numpy(), d[f"{pre}greedy{it}"], err_msg=f"{pre}greedy{it}")
        info = orc.update(s)
        np.testing.assert_allclose([info[f"shared/{k}"] for k in FIX_INFO_KEYS], d[pre + "infos"][it], rtol=1e-5,
                                   atol=1e-7, err_msg=f"{pre}it{it}")
        got = np.concatenate([v.numpy().reshape(-1) for v in orc.m.state_dict().values()])
        np.testing.assert_allclose(got, d[f"{pre}after{it}"], rtol=1e-5, atol=1e-5, err_msg=f"{pre}after{it}")

"""CPU tests of DCG / DCG_S: the float64 kernel restatements (tests/dcg_refs.py) against the reference formulas under
float64 autograd and by hand, the graph edge lists, the K9C argument checks, the shipped configs, the registries and the
out-of-scope errors, a strict state_dict round trip between the oracle and the product's parameter names, and ptxas on
the new kernels."""
import os
import re
import shutil
import subprocess
from argparse import Namespace

import numpy as np
import pytest
import torch

import dcg_refs as R
from oracle_dcg import reference_greedy
from xuance_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = build._nvcc()


def test_graph_edge_lists_match_the_reference_construction():
    from xuance_b200.torch.rl_models import Coordination_Graph
    # coordination_graph.py:122-134, written out for n = 4
    want = {"FULL": [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)], "CYCLE": [(0, 1), (1, 2), (2, 3), (3, 0)],
            "LINE": [(0, 1), (1, 2), (2, 3)], "STAR": [(0, 1), (0, 2), (0, 3)], "VDN": []}
    for graph_type, edges in want.items():
        g = Coordination_Graph(4, graph_type, "cpu")
        g.set_coordination_graph()
        assert g.edges == edges == R.graph_edges(4, graph_type)
        assert g.edges_from.dtype == torch.int32 and g.edges_from.tolist() == [e[0] for e in edges]
        assert g.edges_to.tolist() == [e[1] for e in edges] and g.n_edges == len(edges)
    for n in (1, 2, 3, 5, 8, 25):
        assert len(R.graph_edges(n, "FULL")) == n * (n - 1) // 2 and len(R.graph_edges(n, "CYCLE")) == n
    assert R.graph_edges(1, "CYCLE") == [(0, 0)]                       # a self-loop, as the reference builds it
    with pytest.raises(AttributeError, match="TREE"):
        Coordination_Graph(3, "TREE")


@pytest.mark.parametrize("graph", ["FULL", "CYCLE", "STAR", "VDN"])
@pytest.mark.parametrize("n,A", [(1, 1), (3, 1), (4, 6), (5, 12)])
@pytest.mark.parametrize("use_payoff", [True, False])
def test_q_and_scatter_refs_match_float64_autograd(graph, n, A, use_payoff):
    rng = np.random.default_rng(n * 10 + A)
    edges = R.graph_edges(n, graph)
    Rn = 9
    f = torch.from_numpy(rng.normal(size=(Rn, n, A)).astype(np.float32))
    pay = torch.from_numpy(rng.normal(size=(2, Rn, len(edges), A * A)).astype(np.float32))
    acts = torch.from_numpy(rng.integers(0, A, (Rn, n)))
    q, gf, gp = R.q_autograd(f, pay, edges, acts, use_payoff)
    np.testing.assert_allclose(R.q_ref(f, pay, edges, acts, use_payoff).numpy(), q.numpy(), rtol=1e-14, atol=1e-15)
    df, dp = R.q_bwd_ref(torch.ones(Rn, dtype=torch.float64), acts, edges, n, A, use_payoff)
    assert torch.equal(df, gf)                                           # float(dq/n): one value per agent
    if use_payoff and edges:
        assert torch.equal(dp, gp)                                       # float(dq/E)/2 into both orientations
    else:
        assert gp is None or not gp.any()


@pytest.mark.parametrize("graph", ["FULL", "CYCLE", "LINE", "STAR", "VDN"])
@pytest.mark.parametrize("n,A", [(1, 1), (2, 2), (3, 9), (5, 12), (8, 5)])
@pytest.mark.parametrize("n_iter,normalize", [(0, True), (1, False), (8, True), (8, False)])
def test_greedy_ref_matches_the_reference_loop(graph, n, A, n_iter, normalize):
    rng = np.random.default_rng(n * 7 + A + n_iter)
    edges = R.graph_edges(n, graph)
    Rn = 16
    f = torch.from_numpy(rng.normal(size=(Rn, n, A)).astype(np.float32))
    pay = torch.from_numpy(rng.normal(size=(2, Rn, len(edges), A * A)).astype(np.float32))
    avail = torch.from_numpy((rng.random((Rn, n, A)) < 0.6).astype(np.uint8))
    avail[..., 0] = 1
    a, U = R.greedy_ref(f, pay, edges, n_iter, normalize, avail)
    wa, wU = reference_greedy(f, pay, edges, n_iter, normalize, avail)
    np.testing.assert_allclose(U.numpy(), wU.numpy(), rtol=1e-12, atol=1e-14)
    top2 = torch.where(avail != 0, wU, torch.tensor(-1e10, dtype=torch.float64)).topk(min(2, A), dim=-1).values
    clear = (top2[..., 0] - top2[..., -1] > 1e-9) if A > 1 else torch.ones(Rn, n, dtype=torch.bool)
    assert torch.equal(a[clear], wa[clear])


def test_greedy_ref_ties_masks_and_edge_cases():
    # ties: the first maximal index; all-masked-but-one rows pick the available action
    f = torch.zeros(1, 2, 4)
    pay = torch.zeros(2, 1, 1, 16)
    a, U = R.greedy_ref(f, pay, [(0, 1)], 8, True)
    assert a.tolist() == [[0, 0]] and not U.any()
    avail = torch.zeros(1, 2, 4, dtype=torch.uint8)
    avail[0, 0, 3] = avail[0, 1, 2] = 1
    a, _ = R.greedy_ref(f, pay, [(0, 1)], 8, True, avail)
    assert a.tolist() == [[3, 2]]
    # E = 0 and 0 iterations: U = f / n
    f = torch.arange(6, dtype=torch.float32).reshape(1, 2, 3)
    for edges, it in (([], 8), ([(0, 1)], 0)):
        a, U = R.greedy_ref(f, torch.zeros(2, 1, len(edges), 9), edges, it, True)
        assert torch.equal(U, f.double() / 2) and a.tolist() == [[2, 2]]
    # a payoff that rewards coordinating on action 1 overrides utilities that prefer 0
    f = torch.tensor([[[0.2, 0.0], [0.2, 0.0]]])
    pay = torch.zeros(2, 1, 1, 4)
    pay[:, 0, 0, 3] = 4.0
    a, _ = R.greedy_ref(f, pay, [(0, 1)], 4, False)
    assert a.tolist() == [[1, 1]]


def test_td_ref_matches_float64_autograd():
    rng = np.random.default_rng(2)
    B, n, T = 4, 3, 6
    qe, qn = torch.from_numpy(rng.normal(size=B * T)), torch.from_numpy(rng.normal(size=B * T))
    v, vn = (torch.from_numpy(rng.normal(size=B * T).astype(np.float32)) for _ in range(2))
    rewards = torch.from_numpy(rng.normal(size=(B, n, T)).astype(np.float32))
    terminals = torch.from_numpy((rng.random((B, n, T)) < 0.4).astype(np.float32))
    filled = torch.ones(B, T)
    filled[:, 4:] = 0
    for with_v in (False, True):
        q = qe.clone().requires_grad_(True)
        vv = v.clone().requires_grad_(True)
        Q = q + vv if with_v else q
        Qn = qn + vn if with_v else qn
        y = rewards.mean(dim=1).reshape(-1) + (1 - (terminals != 0).all(dim=1).float().reshape(-1)) * 0.99 * Qn
        f = filled.reshape(-1)
        td = (Q - y.detach()) * f
        loss = (td ** 2).sum() / f.sum()
        loss.backward()
        dq, dv, stats = R.td_ref(qe, qn, v if with_v else None, vn if with_v else None, rewards, terminals, filled,
                                 filled.sum(), 0.99, B * T)
        np.testing.assert_allclose(dq.numpy(), q.grad.numpy(), rtol=1e-13, atol=1e-16)
        np.testing.assert_allclose(stats.numpy(), [loss.item(), Q.mean().item()], rtol=1e-12)
        if with_v:
            assert torch.equal(dv, vv.grad)
        assert (dq.reshape(B, T)[:, 4:] == 0).all()


def test_oracle_and_product_share_parameter_names():
    """A state_dict loads strictly between the product's DeepCoordinationGraph and the oracle (the reference's names)."""
    from oracle_dcg import DCGModelOracle
    from xuance_b200.torch.rl_models import DCG_Utility, DCG_Payoff
    om = DCGModelOracle(3, 12, 7, 10, 16, 16, 16, 16)
    names = list(om.state_dict())
    assert names[0] == "representation.shared.obs_representation.mlp.0.weight"
    assert "bias.values.2.weight" in names and "target_payoffs.output.2.bias" in names
    assert list(DCG_Utility(16, 16, 7).state_dict()) == ["output.0.weight", "output.0.bias", "output.2.weight",
                                                         "output.2.bias"]
    assert DCG_Payoff(32, 16, 7, False, 5).output[2].out_features == 49
    assert DCG_Payoff(32, 16, 7, True, 5).output[2].out_features == 70


def test_low_rank_payoff_is_the_sum_of_outer_products():
    from xuance_b200.torch.rl_models import DCG_Payoff
    torch.manual_seed(0)
    p = DCG_Payoff(8, 8, 4, True, 3)
    x = torch.randn(2, 5, 8)
    out = p(x)
    raw = p.output(x).reshape(2, 5, 3, 2, 4)
    want = sum(torch.outer(raw[1, 4, k, 0], raw[1, 4, k, 1]).reshape(-1) for k in range(3))
    np.testing.assert_allclose(out[1, 4].detach().numpy(), want.detach().numpy(), rtol=1e-6, atol=1e-6)


def test_argument_checks_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    EINVAL, ERANGE = -1, -3
    j = 256  # any non-NULL pointer: validation returns before the device is touched
    g = lambda **k: lib.xb_dcg_greedy(j, k.get("pay", j), k.get("ld", 1 << 30), j, j, k.get("avail"), k.get("ald", 0),
                                      k.get("B", 4), k.get("T", 6), k.get("T1", 7), k.get("t0", 1), k.get("n", 5),
                                      k.get("A", 12), k.get("E", 10), 8, 1, k.get("acts", j), None, None)
    assert g(B=0) == EINVAL and g(n=0) == EINVAL and g(A=0) == EINVAL and g(E=-1) == EINVAL
    assert g(acts=None) == EINVAL and g(pay=None) == EINVAL and g(ld=7) == EINVAL
    assert g(T1=6) == EINVAL                                              # steps t0 .. t0+T-1 must lie inside T1
    assert g(avail=j, ald=11) == EINVAL
    assert g(n=33) == ERANGE and g(A=65) == ERANGE and g(E=513) == ERANGE
    assert g(n=25, A=64, E=300) == ERANGE                                 # the greedy's shared memory
    q = lambda **k: lib.xb_dcg_q_fwd(j, j, 1 << 30, j, j, 1 << 30, j, k.get("greedy", j), j, j, j, 4, k.get("n", 5), 6,
                                     12, 10, 1, j, j, j, j, None)
    assert q(greedy=None) == EINVAL and q(n=33) == ERANGE
    td = lambda **k: lib.xb_dcg_td_fwd_bwd(j, j, k.get("v"), k.get("vn"), j, j, j, j, 4, 5, 6, 0.99,
                                           k.get("rows", 24), j, k.get("dv"), j, j, None)
    assert td(rows=23) == EINVAL                                          # rows_total is the global B*T
    assert td(v=j) == EINVAL and td(v=j, vn=j) == EINVAL                  # V(s), V(s') and dV come together
    bwd = lambda **k: lib.xb_dcg_q_bwd(j, j, j, j, 4, 5, 6, 12, 10, 1, k.get("df", j), k.get("dp", j),
                                       k.get("ld", 1 << 30), None)
    assert bwd(df=None) == EINVAL and bwd(dp=None) == EINVAL and bwd(ld=5) == EINVAL


def _cfg(**over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("dcg", "sc2", "5m_vs_6m")
    cfg.device = "cpu"
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def test_shipped_configs_and_registries():
    import yaml
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    for env_id in ("5m_vs_6m", "3m"):
        cfg = get_arguments("dcg", "sc2", env_id)
        assert cfg.env_id == env_id and cfg.agent == "DCG" and cfg.learner == "DCG_Learner"
        assert cfg.graph_type == "FULL" and cfg.n_msg_iterations == 8 and cfg.msg_normalized is True
        assert cfg.hidden_utility_dim == 64 and cfg.hidden_payoff_dim == 64 and cfg.low_rank_payoff is False
        assert cfg.payoff_rank == 5 and cfg.use_rnn and cfg.use_actions_mask and cfg.sync_frequency == 200
    assert REGISTRY_Agents["DCG"] is REGISTRY_Agents["DCG_S"]
    assert REGISTRY_Agents["DCG"].__name__ == "DCG_Agents"
    assert REGISTRY_Learners["DCG_Learner"].__name__ == "DCG_Learner"
    root = os.path.join(ROOT, "xuance_b200")
    src = "".join(open(os.path.join(root, *f.split("/"))).read() for f in
                  ("torch/agents/marl.py", "torch/agents/dcg_agents.py", "torch/learners/qmix_learner.py",
                   "torch/learners/dcg_learner.py", "torch/agents/agent.py", "torch/learners/learner.py"))
    hard = set(re.findall(r"(?<![a-zA-Z_])(?:self\.)?(?:config|cfg)\.([a-zA-Z_][a-zA-Z0-9_]*)\b(?!\s*=[^=])", src))
    soft = set(re.findall(r"(?:getattr|hasattr)\((?:self\.)?config,\s*.([a-zA-Z_0-9]+).", src))
    base = set(yaml.safe_load(open(os.path.join(root, "configs", "basic.yaml"))))
    base |= {"hidden_dim_mixing_net", "hidden_dim_hyper_net"}            # QMIX_Agents' mixer (marl.py), not DCG's
    for env_id in ("5m_vs_6m", "3m"):
        y = yaml.safe_load(open(os.path.join(root, "configs", "dcg", "sc2", f"{env_id}.yaml")))
        assert not sorted(hard - soft - base - set(y)), env_id


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import REGISTRY_Agents

    def kw(n=3, A=7):
        keys = [f"agent_{i}" for i in range(n)]
        return dict(num_agents=n, agent_keys=keys, state_space=Box(-1, 1, (10,), np.float32),
                    observation_space={k: Box(-1, 1, (12,), np.float32) for k in keys},
                    action_space={k: Discrete(A) for k in keys})
    with pytest.raises(NotImplementedError, match="use_rnn"):
        REGISTRY_Agents["DCG"](_cfg(use_rnn=False), **kw())
    with pytest.raises(NotImplementedError, match="use_parameter_sharing"):
        REGISTRY_Agents["DCG_S"](_cfg(agent="DCG_S", use_parameter_sharing=False), **kw())
    with pytest.raises(NotImplementedError, match="LSTM"):
        REGISTRY_Agents["DCG"](_cfg(rnn="LSTM"), **kw())
    with pytest.raises(NotImplementedError, match="outside the supported"):
        REGISTRY_Agents["DCG"](_cfg(), **kw(n=33))
    with pytest.raises(NotImplementedError, match="outside the supported"):
        REGISTRY_Agents["DCG"](_cfg(), **kw(n=5, A=65))
    with pytest.raises(NotImplementedError, match="outside the supported"):
        REGISTRY_Agents["DCG"](_cfg(), **kw(n=25, A=64))                  # 300 edges: the greedy's shared memory
    with pytest.raises(AttributeError, match="graph type"):
        REGISTRY_Agents["DCG"](_cfg(graph_type="TREE"), **kw())


def test_learner_refuses_unknown_agents_and_feed_forward_agents():
    from xuance_b200.torch.learners import DCG_Learner
    with pytest.raises(AttributeError, match="QTRAN"):
        DCG_Learner(Namespace(agent="QTRAN", use_rnn=True), None, None, None)
    with pytest.raises(NotImplementedError, match="use_rnn"):
        DCG_Learner(Namespace(agent="DCG", use_rnn=False), None, None, None)


@pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not available")
def test_dcg_kernels_compile_without_spills(tmp_path):
    flags = [f for f in build.NVCC_FLAGS if f not in ("--use_fast_math=false", "-shared")]
    cmd = [NVCC] + flags + ["-c", os.path.join(build.CSRC, "dcg.cu"), "-o", str(tmp_path / "dcg.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S*dcg\S*)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = sum(int(x) for x in m.groups())
            cur = None
    assert len(kernels) == 5, log                                        # the greedy with and without the F_e table
    assert {k: v for k, v in kernels.items() if v} == {}


# ---------------------------------------------------------------- the reference fixture (tests/golden/dcg_update.npz)
GOLDEN = os.path.join(ROOT, "tests", "golden", "dcg_update.npz")
# (name, agent, graph_type, msg_normalized, low_rank_payoff, n_msg_iterations), as make_golden_dcg.py records them
FIX_CASES = [("dcg_full", "DCG", "FULL", True, False, 8), ("dcg_s_full", "DCG_S", "FULL", True, False, 8),
             ("dcg_cycle_raw", "DCG", "CYCLE", False, False, 8), ("dcg_s_cycle_lowrank", "DCG_S", "CYCLE", True, True, 4),
             ("dcg_iter0", "DCG", "FULL", True, False, 0), ("dcg_s_iter0", "DCG_S", "FULL", True, False, 0),
             ("dcg_s_vdn", "DCG_S", "VDN", True, False, 8)]
FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_HID, FIX_RANK = 4, 12, 6, 10, 16, 3
FIX_UPDATES, FIX_SNAPSHOTS = 4, (1, 3)
FIX_INFO_KEYS = ("loss_Q", "predictQ", "learning_rate")


def fixture_init(d, name):
    pre = name + "/init/"
    return {k[len(pre):]: torch.from_numpy(d[k]) for k in d.files if k.startswith(pre)}


def fixture_sample(d, name, it, keys):
    p = f"{name}/in{it}/"
    s = {f: {k: d[p + f][:, i] for i, k in enumerate(keys)}
         for f in ("obs", "actions", "rewards", "terminals", "agent_mask", "avail_actions")}
    B, T = d[p + "filled"].shape
    s.update(filled=d[p + "filled"], state=d[p + "state"], batch_size=B, sequence_length=T)
    return s


@pytest.mark.parametrize("case", FIX_CASES, ids=[c[0] for c in FIX_CASES])
def test_oracle_reproduces_the_reference_fixture(case):
    from oracle_dcg import DCGModelOracle, DCGLearnerOracle
    name, agent, graph, normalized, low_rank, n_iter = case
    d = np.load(GOLDEN)
    keys = [f"agent_{i}" for i in range(FIX_N)]
    om = DCGModelOracle(FIX_N, FIX_OBS, FIX_A, FIX_S if agent == "DCG_S" else None, FIX_HID, FIX_HID, FIX_HID, FIX_HID,
                        low_rank, FIX_RANK)
    om.load_state_dict(fixture_init(d, name), strict=True)              # the reference's parameter names
    orc = DCGLearnerOracle(om, keys, R.graph_edges(FIX_N, graph), n_iter, normalized, sync_frequency=2,
                           end_factor_lr_decay=0.5, total_iters=int(d[name + "/total_iters"]))
    for it in range(FIX_UPDATES):
        info = orc.update(fixture_sample(d, name, it, keys))
        np.testing.assert_allclose([info[k] for k in FIX_INFO_KEYS], d[name + "/infos"][it], rtol=2e-6, atol=1e-7)
        if it in FIX_SNAPSHOTS:
            got = np.concatenate([v.numpy().reshape(-1) for v in om.state_dict().values()])
            np.testing.assert_allclose(got, d[f"{name}/after{it}"], rtol=1e-5, atol=1e-6)
    if agent == "DCG_S" and (graph == "VDN" or n_iter == 0):       # no payoffs: V(s) is not in Q, the bias never moves
        init = fixture_init(d, name)
        for k, v in om.state_dict().items():
            if k.startswith("bias."):
                assert torch.equal(v, init[k]), k


@pytest.mark.parametrize("graph", ["FULL", "CYCLE", "LINE", "STAR", "VDN"])
def test_greedy_ref_reproduces_the_reference_act(graph):
    d = np.load(GOLDEN)
    pre = f"act/{graph}/"
    f, pay, avail, edges = fixture_act_heads(d, graph)
    a, U = R.greedy_ref(f, pay, edges, 8, True, avail)
    wU, wa = torch.from_numpy(d[pre + "U"]), torch.from_numpy(d[pre + "actions"])
    np.testing.assert_allclose(U.numpy(), wU.numpy(), rtol=1e-12, atol=1e-14)
    clear = fixture_clear_rows(wU, avail)
    assert clear.float().mean() > 0.9 and torch.equal(a[clear], wa[clear])


def fixture_act_heads(d, graph):
    """The recorded act() inputs through the recorded utility / payoff heads: f [R, n, A], pay [2, R, E, A*A]."""
    pre = f"act/{graph}/"
    w = lambda k: torch.from_numpy(d[pre + k])
    h = w("hidden")
    mlp = lambda x, m: torch.relu(x @ w(m + ".output.0.weight").T + w(m + ".output.0.bias")) @ \
        w(m + ".output.2.weight").T + w(m + ".output.2.bias")
    edges = R.graph_edges(h.shape[1], graph)
    fr = torch.tensor([e[0] for e in edges], dtype=torch.long)
    to = torch.tensor([e[1] for e in edges], dtype=torch.long)
    x = torch.stack([torch.cat([h[:, fr], h[:, to]], -1), torch.cat([h[:, to], h[:, fr]], -1)])
    return mlp(h, "utility"), mlp(x, "payoffs"), w("avail"), edges


def fixture_clear_rows(U, avail):
    """Agents whose two best available U values differ by more than 1e-9 (the arg-max is then decided)."""
    top2 = torch.where(avail != 0, U, torch.tensor(-1e10, dtype=torch.float64)).topk(2, dim=-1).values
    return top2[..., 0] - top2[..., 1] > 1e-9

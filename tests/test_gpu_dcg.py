"""GPU tests of DCG / DCG_S: the K9C kernels against the float64 restatements (tests/dcg_refs.py), bit for bit; shards
and launch-to-launch identity; DCG_Learner against the torch-CPU oracle (tests/oracle_dcg.py), eager and graphed;
graphed equals eager; the acting greedy equals the learner-side greedy; checkpoints; and both variants learning through
REGISTRY_Agents."""
from argparse import Namespace

import numpy as np
import pytest
import torch

import dcg_refs as R
import test_dcg as T
from oracle_dcg import DCGModelOracle, DCGLearnerOracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GRAPHS = ("FULL", "CYCLE", "LINE", "STAR", "VDN")


def _edges_dev(edges):
    fr = torch.tensor([e[0] for e in edges], dtype=torch.int32, device=DEV)
    to = torch.tensor([e[1] for e in edges], dtype=torch.int32, device=DEV)
    return fr, to


def _run_greedy(f, pay, edges, n_iter, normalize, avail=None):
    """f [R, n, A], pay [2, R, E, A*A], avail [R, n, A] on the CPU -> (actions, U, return code) from the kernel."""
    from xuance_b200 import _lib
    Rn, n, A = f.shape
    E = len(edges)
    fd = f.reshape(Rn, n, 1, A).to(DEV).contiguous()
    pd = pay.to(DEV).contiguous() if E else None
    ad = avail.reshape(Rn, n, 1, A).to(DEV).to(torch.uint8).contiguous() if avail is not None else None
    fr, to = _edges_dev(edges)
    acts = torch.empty(Rn, n, dtype=torch.int32, device=DEV)
    U = torch.empty(Rn, n, A, dtype=torch.float64, device=DEV)
    lib = _lib.load()
    rc = lib.xb_dcg_greedy(_lib.ptr(fd), _lib.ptr(pd), pd[0].numel() if E else 0, _lib.ptr(fr), _lib.ptr(to),
                           _lib.ptr(ad), A if ad is not None else 0, Rn, 1, 1, 0, n, A, E, n_iter, int(normalize),
                           _lib.ptr(acts), _lib.ptr(U), None)
    torch.cuda.synchronize()
    return acts.cpu(), U.cpu(), rc


def _greedy_inputs(rng, Rn, n, A, E, masked):
    f = R.quantised(rng, (Rn, n, A))
    pay = R.quantised(rng, (2, Rn, E, A * A))
    avail = None
    if masked:
        avail = torch.from_numpy((rng.random((Rn, n, A)) < 0.6).astype(np.uint8))
        avail[..., -1] = 1
    return f, pay, avail


SHAPES = [(1, 1), (2, 2), (3, 9), (5, 12), (8, 31), (8, 64), (25, 12), (25, 2)]   # (n, A)


@pytest.mark.parametrize("graph", GRAPHS)
@pytest.mark.parametrize("n,A", SHAPES)
def test_greedy_matches_float64_bit_for_bit(graph, n, A):
    edges = R.graph_edges(n, graph)
    rng = np.random.default_rng(n * 100 + A + len(graph))
    for Rn in (1, 2, 31, 32, 33, 1920):
        if Rn == 1920 and n * A > 100:
            continue
        f, pay, avail = _greedy_inputs(rng, Rn, n, A, len(edges), Rn % 2 == 1)
        for n_iter in (0, 1, 8):
            for normalize in (False, True):
                got_a, got_U, rc = _run_greedy(f, pay, edges, n_iter, normalize, avail)
                assert rc == 0
                want_a, want_U = R.greedy_ref(f, pay, edges, n_iter, normalize, avail)
                assert torch.equal(got_U, want_U), (Rn, n_iter, normalize)
                assert torch.equal(got_a.long(), want_a), (Rn, n_iter, normalize)


def test_greedy_at_the_largest_instance_count():
    rng = np.random.default_rng(7)
    edges = R.graph_edges(5, "FULL")
    f, pay, avail = _greedy_inputs(rng, 2 ** 17 + 3, 5, 12, len(edges), True)
    got_a, got_U, rc = _run_greedy(f, pay, edges, 8, True, avail)
    assert rc == 0
    want_a, want_U = R.greedy_ref(f, pay, edges, 8, True, avail)
    assert torch.equal(got_U, want_U) and torch.equal(got_a.long(), want_a)


def _q_inputs(rng, B, n, T, A, E):
    f = lambda: R.quantised(rng, (B, n, T + 1, A), 1 / 64)
    p = lambda: R.quantised(rng, (2, B, E, T + 1, A * A), 1 / 64)
    actions = torch.from_numpy(rng.integers(0, A, (B, n, T)).astype(np.float32))
    greedy = torch.from_numpy(rng.integers(0, A, (B * T, n)).astype(np.int32))
    filled = torch.from_numpy((rng.random((B, T)) < 0.8).astype(np.float32))
    return f(), p(), f(), p(), actions, greedy, filled


def _run_q(f_e, p_e, f_t, p_t, actions, greedy, filled, edges, use_payoff):
    from xuance_b200 import _lib
    B, n, T1, A = f_e.shape
    T, E = T1 - 1, len(edges)
    d = [x.to(DEV).contiguous() for x in (f_e, p_e, f_t, p_t, actions, greedy, filled)]
    fr, to = _edges_dev(edges)
    qe, qn = torch.empty(B * T, dtype=torch.float64, device=DEV), torch.empty(B * T, dtype=torch.float64, device=DEV)
    fs = torch.empty(1, device=DEV)
    _lib.call("xb_dcg_q_fwd", _lib.ptr(d[0]), _lib.ptr(d[1]), d[1][0].numel(), _lib.ptr(d[2]), _lib.ptr(d[3]),
              d[3][0].numel(), _lib.ptr(d[4]), _lib.ptr(d[5]), _lib.ptr(d[6]), _lib.ptr(fr), _lib.ptr(to), B, n, T, A,
              E, int(use_payoff), _lib.ptr(qe), _lib.ptr(qn), _lib.ptr(fs), _lib.ptr(_lib.scratch(DEV)))
    torch.cuda.synchronize()
    return qe.cpu(), qn.cpu(), fs.cpu()


def _rows(x, t0, T):
    """[B, n, T+1, K] (or [2, B, E, T+1, K]) -> the instances at steps t0..t0+T-1 as [B*T, n, K] ([2, B*T, E, K])."""
    if x.dim() == 4:
        return x[:, :, t0:t0 + T].transpose(1, 2).reshape(-1, x.shape[1], x.shape[3])
    return x[:, :, :, t0:t0 + T].transpose(2, 3).reshape(2, x.shape[1] * T, x.shape[2], x.shape[4])


@pytest.mark.parametrize("graph,n,A,use_payoff", [("FULL", 5, 12, True), ("CYCLE", 3, 9, True), ("FULL", 5, 12, False),
                                                  ("VDN", 4, 7, True), ("STAR", 1, 1, True), ("LINE", 8, 33, True)])
@pytest.mark.parametrize("B,T", [(1, 1), (3, 17), (32, 60)])
def test_q_td_and_scatter_match_float64(graph, n, A, use_payoff, B, T):
    from xuance_b200 import _lib
    rng = np.random.default_rng(B * 31 + T + n)
    edges = R.graph_edges(n, graph)
    E = len(edges)
    f_e, p_e, f_t, p_t, actions, greedy, filled = _q_inputs(rng, B, n, T, A, E)
    qe, qn, fs = _run_q(f_e, p_e, f_t, p_t, actions, greedy, filled, edges, use_payoff)
    acts = actions.transpose(1, 2).reshape(B * T, n)
    assert torch.equal(qe, R.q_ref(_rows(f_e, 0, T), _rows(p_e, 0, T), edges, acts, use_payoff))
    assert torch.equal(qn, R.q_ref(_rows(f_t, 1, T), _rows(p_t, 1, T), edges, greedy.long(), use_payoff))
    assert float(fs) == float(filled.sum())
    if float(fs) == 0:
        return
    rewards = torch.from_numpy(rng.normal(size=(B, n, T)).astype(np.float32))
    terminals = torch.from_numpy((rng.random((B, n, T)) < 0.3).astype(np.float32))
    for dcg_s in (False, True):
        v = torch.from_numpy(rng.normal(size=B * T).astype(np.float32)) if dcg_s else None
        vn = torch.from_numpy(rng.normal(size=B * T).astype(np.float32)) if dcg_s else None
        dq = torch.empty(B * T, dtype=torch.float64, device=DEV)
        dv = torch.empty(B * T, device=DEV) if dcg_s else None
        stats = torch.empty(2, device=DEV)
        ins = [None if x is None else x.to(DEV).contiguous() for x in (qe, qn, v, vn, rewards, terminals, filled, fs)]
        _lib.call("xb_dcg_td_fwd_bwd", *[_lib.ptr(x) for x in ins], B, n, T, 0.99, B * T, _lib.ptr(dq), _lib.ptr(dv),
                  _lib.ptr(stats), _lib.ptr(_lib.scratch(DEV)))
        torch.cuda.synchronize()
        w_dq, w_dv, w_st = R.td_ref(qe, qn, v, vn, rewards, terminals, filled, fs, 0.99, B * T)
        assert torch.equal(dq.cpu(), w_dq)
        if dcg_s:
            assert torch.equal(dv.cpu(), w_dv)
        np.testing.assert_allclose(stats.cpu().numpy(), w_st.numpy(), rtol=1e-6, atol=1e-7)
    # the scatter, bit for bit, into pre-zeroed outputs
    dq = torch.from_numpy(rng.normal(size=B * T))
    df = torch.zeros(B, n, T + 1, A, device=DEV)
    dp = torch.zeros(2, B, E, T + 1, A * A, device=DEV)
    fr, to = _edges_dev(edges)
    dqd, ad = dq.to(DEV), actions.to(DEV)
    _lib.call("xb_dcg_q_bwd", _lib.ptr(dqd), _lib.ptr(ad), _lib.ptr(fr), _lib.ptr(to), B, n, T, A, E, int(use_payoff),
              _lib.ptr(df), _lib.ptr(dp), dp[0].numel())
    torch.cuda.synchronize()
    w_df, w_dp = R.q_bwd_ref(dq, acts, edges, n, A, use_payoff)
    assert torch.equal(_rows(df.cpu(), 0, T), w_df) and (df[:, :, T] == 0).all()
    assert torch.equal(_rows(dp.cpu(), 0, T), w_dp) and (dp[:, :, :, T] == 0).all()


@pytest.mark.parametrize("G", [2, 3, 8])
def test_td_shards_sum_to_the_full_batch(G):
    from xuance_b200 import _lib
    rng = np.random.default_rng(G)
    B, n, T = 48, 5, 60
    qe, qn = torch.from_numpy(rng.normal(size=B * T)), torch.from_numpy(rng.normal(size=B * T))
    rewards = torch.from_numpy(rng.normal(size=(B, n, T)).astype(np.float32))
    terminals = torch.from_numpy((rng.random((B, n, T)) < 0.2).astype(np.float32))
    filled = torch.from_numpy((rng.random((B, T)) < 0.8).astype(np.float32))
    fs = filled.sum().reshape(1)

    def run(rows, b):
        dq, stats = torch.empty(len(rows), dtype=torch.float64, device=DEV), torch.empty(2, device=DEV)
        ins = [x.to(DEV).contiguous() for x in (qe[rows], qn[rows], rewards[b], terminals[b], filled[b], fs)]
        _lib.call("xb_dcg_td_fwd_bwd", _lib.ptr(ins[0]), _lib.ptr(ins[1]), None, None, *[_lib.ptr(x) for x in ins[2:]],
                  len(b), n, T, 0.99, B * T, _lib.ptr(dq), None, _lib.ptr(stats), _lib.ptr(_lib.scratch(DEV)))
        torch.cuda.synchronize()
        return dq.cpu(), stats.cpu()

    full = run(torch.arange(B * T), torch.arange(B))
    parts = []
    for idx in np.array_split(np.arange(B), G):
        rows = torch.from_numpy((idx[:, None] * T + np.arange(T)[None]).reshape(-1))
        parts.append(run(rows, torch.from_numpy(idx)))
    assert torch.equal(torch.cat([p[0] for p in parts]), full[0])
    np.testing.assert_allclose(sum(p[1].double() for p in parts).numpy(), full[1].numpy(), rtol=2e-6, atol=1e-7)


def test_launch_to_launch_bit_identity():
    rng = np.random.default_rng(5)
    edges = R.graph_edges(5, "FULL")
    f, pay, avail = _greedy_inputs(rng, 1920, 5, 12, len(edges), True)
    a, b = _run_greedy(f, pay, edges, 8, True, avail), _run_greedy(f, pay, edges, 8, True, avail)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    ins = _q_inputs(rng, 32, 5, 60, 12, len(edges))
    x, y = _run_q(*ins, edges, True), _run_q(*ins, edges, True)
    assert all(torch.equal(p, q) for p, q in zip(x, y))


# ---------------------------------------------------------------- model, learner, agents
def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _product_model(n, obs_dim, A, S=None, hid=64, graph="FULL", n_iter=8, normalize=True, low_rank=False, rank=1):
    import torch.nn as nn
    from xuance_b200.common import AgentGrouping, Discrete
    from xuance_b200.torch.rl_models import (AgentFeatureEncoder, Basic_RNN_K13, ValueHead, DCG_Utility, DCG_Payoff,
                                             Coordination_Graph, DeepCoordinationGraph)
    keys = [f"agent_{i}" for i in range(n)]
    rep = Basic_RNN_K13(input_shape=(obs_dim,), initialize=nn.init.orthogonal_, activation=nn.ReLU, device=DEV,
                        fc_hidden_sizes=[hid], recurrent_hidden_size=hid)
    g = Coordination_Graph(n, graph, DEV)
    g.set_coordination_graph()
    bias = ValueHead(S, [hid], None, nn.init.orthogonal_, nn.ReLU, DEV) if S else None
    grouping = AgentGrouping.shared(keys)
    model = DeepCoordinationGraph(grouping, {k: Discrete(A) for k in keys}, nn.ModuleDict({'shared': AgentFeatureEncoder(rep)}),
                                  DCG_Utility(hid, hid, A, DEV), DCG_Payoff(2 * hid, hid, A, low_rank, rank, DEV), g,
                                  dcg_s=S is not None, bias=bias, use_rnn=True, device=DEV, n_msg_iterations=n_iter,
                                  msg_normalized=normalize).to(DEV)
    return keys, grouping, model


def _learner(grouping, model, **over):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import DCG_Learner
    cfg = dict(device=DEV, model_dir="/tmp/xb200_dcg_models", use_cuda_graph=False, use_grad_clip=False,
               grad_clip_norm=0.5, parallels=4, running_steps=100000, start_training=0, use_rnn=True,
               use_actions_mask=True, learning_rate=7e-4, sync_frequency=2, gamma=0.99, end_factor_lr_decay=0.5,
               use_linear_lr_decay=True, agent="DCG")
    cfg.update(over)
    return DCG_Learner(Namespace(**cfg), grouping, model, BaseCallback())


def _sample(rng, keys, B, T, obs_dim, A, S):
    from wqmix_refs import fix_sample
    return fix_sample(rng, keys, B=B, T=T, obs_dim=obs_dim, A=A, S=S or 4)


CASES = [("DCG", "FULL", 8, True, False), ("DCG_S", "FULL", 8, True, False), ("DCG", "CYCLE", 8, False, False),
         ("DCG_S", "CYCLE", 4, True, True), ("DCG", "FULL", 0, True, False), ("DCG", "VDN", 8, True, False),
         ("DCG_S", "VDN", 8, True, False)]


def _intended_run(agent, graph, n_iter, normalize, low_rank, use_graph, updates=4, seed=0):
    _no_tf32()
    torch.manual_seed(seed)
    n, obs_dim, A, T, B = 4, 20, 7, 12, 6
    S = 10 if agent == "DCG_S" else None
    keys, grouping, model = _product_model(n, obs_dim, A, S, 32, graph, n_iter, normalize, low_rank, 3)
    om = DCGModelOracle(n, obs_dim, A, S, 32, 32, 32, 32, low_rank, 3)
    model.load_state_dict(om.state_dict(), strict=True)
    lrn = _learner(grouping, model, agent=agent, use_cuda_graph=use_graph, episode_length=T)
    orc = DCGLearnerOracle(om, keys, R.graph_edges(n, graph), n_iter, normalize, sync_frequency=2,
                           end_factor_lr_decay=0.5, total_iters=lrn.total_iters)
    rng = np.random.default_rng(seed + 1)
    infos = []
    for _ in range(updates):
        s = _sample(rng, keys, B, T, obs_dim, A, S)
        infos.append((lrn.update(s), orc.update(s)))
    return model, om, infos


@pytest.mark.parametrize("agent,graph,n_iter,normalize,low_rank", CASES)
@pytest.mark.parametrize("use_graph", [False, True])
def test_learner_matches_the_oracle(agent, graph, n_iter, normalize, low_rank, use_graph):
    model, om, infos = _intended_run(agent, graph, n_iter, normalize, low_rank, use_graph)
    for it, (ip, io) in enumerate(infos):
        for k in ("predictQ", "learning_rate"):
            np.testing.assert_allclose(ip[k], io[k], rtol=5e-4, atol=1e-5, err_msg=f"{k} it{it}")
        # max-plus U values of two actions can tie to within the float32 difference of GPU and CPU heads; the greedy
        # next action of such an agent may then differ, which moves one row's target: looser on the loss alone
        np.testing.assert_allclose(ip["loss_Q"], io["loss_Q"], rtol=5e-3, atol=1e-5, err_msg=f"loss_Q it{it}")
    so, sp = om.state_dict(), model.state_dict()
    for k in so:
        np.testing.assert_allclose(sp[k].cpu().numpy(), so[k].numpy(), rtol=2e-3, atol=3e-4, err_msg=k)


def test_graphed_update_is_bit_equal_to_eager():
    m_e, _, i_e = _intended_run("DCG_S", "FULL", 8, True, False, False, updates=3, seed=4)
    m_g, _, i_g = _intended_run("DCG_S", "FULL", 8, True, False, True, updates=3, seed=4)
    for (a, _), (b, _) in zip(i_e, i_g):
        assert a == b
    for (k, v), (_, w) in zip(m_e.state_dict().items(), m_g.state_dict().items()):
        assert torch.equal(v, w), k


def test_acting_greedy_equals_the_learner_greedy():
    """One acting step per time step, carrying the GRU state, gives the learner-side greedy on the same hidden states."""
    from xuance_b200.torch.rl_models.dcg import dcg_greedy
    _no_tf32()
    torch.manual_seed(3)
    n, obs_dim, A, T, B = 5, 16, 12, 9, 4
    keys, grouping, model = _product_model(n, obs_dim, A, None, 64, "FULL")
    rng = np.random.default_rng(3)
    obs = torch.from_numpy(rng.normal(size=(B, n, T + 1, obs_dim)).astype(np.float32)).to(DEV)
    avail = torch.from_numpy((rng.random((B, n, T + 1, A)) < 0.6).astype(np.uint8)).to(DEV)
    avail[..., 0] = 1
    with torch.no_grad():
        h = model.hidden_states(obs.flatten(0, 1)).reshape(B, n, T + 1, -1)
        f, pay = model.heads(h)
        want = dcg_greedy(f, pay, model.graph, 8, True, T + 1, 0, avail.contiguous()).reshape(B, T + 1, n)
    rnn = model.init_rnn_states(B)
    for t in range(T + 1):
        acts, _, rnn = model(obs[:, :, t].reshape(B * n, obs_dim), avail[:, :, t].reshape(B * n, A), rnn)
        assert torch.equal(acts.reshape(B, n), want[:, t]), t


def test_checkpoint_round_trip(tmp_path):
    _no_tf32()
    torch.manual_seed(1)
    rng = np.random.default_rng(1)
    keys, grouping, model = _product_model(3, 12, 7, 10, 32)
    lrn = _learner(grouping, model, agent="DCG_S", end_factor_lr_decay=1.0, episode_length=8)
    samples = [_sample(rng, keys, 6, 8, 12, 7, 10) for _ in range(3)]
    for s in samples[:2]:
        lrn.update(s)
    path = str(tmp_path / "dcg.pth")
    lrn.save_model(path)
    _, grouping2, model2 = _product_model(3, 12, 7, 10, 32)
    lrn2 = _learner(grouping2, model2, agent="DCG_S", end_factor_lr_decay=1.0, episode_length=8)
    lrn2.load_model(path)
    lrn2.iterations = lrn.iterations
    for (k, v), (_, w) in zip(model.state_dict().items(), model2.state_dict().items()):
        assert torch.equal(v, w), k
    assert lrn.update(samples[2]) == lrn2.update(samples[2])


def _agent_config(**over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("dcg", "sc2", "3m")
    base = dict(vectorize="Dummy_StarCraft2", parallels=8, buffer_size=64, batch_size=16, learning_rate=2e-3, gamma=0.5,
                start_greedy=1.0, end_greedy=0.05, decay_step_greedy=12000, start_training=200, running_steps=40000,
                n_epochs=4, sync_frequency=20, device=DEV, model_dir="/tmp/xb200_dcg_models",
                log_dir="/tmp/xb200_dcg_logs", episode_limit=20, p_death=0.02, distributed_training=False,
                use_cuda_graph=False)
    base.update(over)
    for k, v in base.items():
        setattr(cfg, k, v)
    return cfg


@pytest.mark.parametrize("agent", ["DCG", "DCG_S"])
def test_dcg_learns_through_the_agent_registry(agent):
    """REGISTRY_Agents["DCG"] / ["DCG_S"] on the cue-following SMAC-shaped env (3m): the greedy team score rises."""
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.rl_models import DeepCoordinationGraph
    cfg = _agent_config(agent=agent)
    envs = make_envs(cfg)
    ag = REGISTRY_Agents[agent](cfg, envs)
    assert isinstance(ag.model, DeepCoordinationGraph) and ag.model.dcg_s == (agent == "DCG_S")
    before = float(np.mean(ag.test(16, make_envs(cfg))))
    info = ag.train(cfg.running_steps // cfg.parallels)
    assert {"loss_Q", "predictQ"} <= set(info) and np.isfinite(info["loss_Q"])
    after = float(np.mean(ag.test(32, make_envs(cfg))))
    assert after > before + 2.0, (before, after)
    ag.finish()


# ---------------------------------------------------------------- against the reference fixture (tests/golden/dcg_update.npz)
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("case", T.FIX_CASES, ids=[c[0] for c in T.FIX_CASES])
def test_learner_reproduces_the_reference_fixture(case, use_graph):
    _no_tf32()
    name, agent, graph, normalized, low_rank, n_iter = case
    d = np.load(T.GOLDEN)
    keys, grouping, model = _product_model(T.FIX_N, T.FIX_OBS, T.FIX_A, T.FIX_S if agent == "DCG_S" else None,
                                           T.FIX_HID, graph, n_iter, normalized, low_rank, T.FIX_RANK)
    init = T.fixture_init(d, name)
    model.load_state_dict(init, strict=True)                   # a reference state_dict loads strictly
    lrn = _learner(grouping, model, agent=agent, use_cuda_graph=use_graph, episode_length=8)
    assert lrn.total_iters == int(d[name + "/total_iters"])
    for it in range(T.FIX_UPDATES):
        info = lrn.update(T.fixture_sample(d, name, it, keys))
        np.testing.assert_allclose([info[k] for k in T.FIX_INFO_KEYS], d[name + "/infos"][it], rtol=2e-4, atol=1e-6,
                                   err_msg=f"{name} it{it}")
        if it in T.FIX_SNAPSHOTS:
            flat = np.concatenate([v.cpu().numpy().reshape(-1) for v in model.state_dict().values()])
            np.testing.assert_allclose(flat, d[f"{name}/after{it}"], rtol=1e-4, atol=2e-5, err_msg=f"{name} after{it}")
    if agent == "DCG_S" and (graph == "VDN" or n_iter == 0):       # no payoffs: V(s) is not in Q, the bias never moves
        for k, v in model.state_dict().items():
            if k.startswith("bias."):
                assert torch.equal(v.cpu(), init[k]), k


@pytest.mark.parametrize("graph", GRAPHS)
def test_greedy_reproduces_the_reference_act(graph):
    """The reference's act() on recorded hidden states: U to 1e-12 relative, equal actions wherever the top two differ
    by more than 1e-9."""
    d = np.load(T.GOLDEN)
    f, pay, avail, edges = T.fixture_act_heads(d, graph)
    a, U, rc = _run_greedy(f.float(), pay.float() if edges else pay, edges, 8, True, avail)
    assert rc == 0
    wU, wa = torch.from_numpy(d[f"act/{graph}/U"]), torch.from_numpy(d[f"act/{graph}/actions"])
    np.testing.assert_allclose(U.numpy(), wU.numpy(), rtol=1e-12, atol=1e-14)
    clear = T.fixture_clear_rows(wU, avail)
    assert torch.equal(a.long()[clear], wa[clear])

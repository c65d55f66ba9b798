"""GPU tests of Weighted QMIX: the K9W kernels against the float64 restatements (tests/wqmix_refs.py), shards, launch-to-
launch identity; WQMIX_Learner against the reference fixture (tests/golden/wqmix_update.npz) and against the oracle's
intended computation, eager and graphed; checkpoints; and OW-QMIX / CW-QMIX learning through REGISTRY_Agents."""
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn as nn

import wqmix_refs as R
from oracle_wqmix import WQMIXModelOracle, WQMIXLearnerOracle
from test_wqmix import GOLDEN, fixture_sample

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _select_inputs(rng, B, n, T, A, masked):
    q = lambda: torch.from_numpy(np.round(rng.normal(size=(B, n, T + 1, A)) * 4) / 4).float()   # coarse: many ties
    actions = torch.from_numpy(rng.integers(0, A, (B, n, T)).astype(np.float32))
    agent_mask = torch.from_numpy((rng.random((B, n, T)) < 0.85).astype(np.float32))
    filled = torch.from_numpy((rng.random((B, T)) < 0.8).astype(np.float32))
    avail = torch.from_numpy((rng.random((B, n, T + 1, A)) < 0.6).astype(np.uint8)) if masked else None
    if masked:
        avail[..., 0] = 1
    return q(), q(), q(), q(), actions, agent_mask, filled, avail


def _run_select(q_all, q_cent, q_cent_tgt, q_tgt, actions, agent_mask, filled, avail, double_q):
    from xuance_b200 import _lib
    B, n, T1, A = q_all.shape
    T = T1 - 1
    c = lambda x: None if x is None else x.to(DEV).contiguous()
    ins = [c(x) for x in (q_all, q_cent, q_cent_tgt, q_tgt, actions, agent_mask, filled, avail)]
    out = [torch.empty(B * T, n, device=DEV) for _ in range(3)]
    greedy = torch.empty(B, n, T, dtype=torch.int32, device=DEV)
    agree = torch.empty(B * T, dtype=torch.uint8, device=DEV)
    fs, scratch = torch.empty(1, device=DEV), _lib.scratch(DEV)
    _lib.call("xb_wqmix_select_fwd", *[_lib.ptr(x) for x in ins], A if avail is not None else 0, B, n, T, A,
              int(double_q), *[_lib.ptr(x) for x in out], _lib.ptr(greedy), _lib.ptr(agree), _lib.ptr(fs),
              _lib.ptr(scratch))
    torch.cuda.synchronize()
    return [x.cpu() for x in out] + [greedy.cpu(), agree.cpu(), fs.cpu()]


def _run_loss(q_tot, q_ff, q_ff_next, rewards, terminals, filled, agree, filled_sum, mode, rows_total, scratch=None):
    from xuance_b200 import _lib
    B, n, T = rewards.shape
    c = lambda x: x.to(DEV).contiguous()
    ins = [c(x) for x in (q_tot, q_ff, q_ff_next, rewards, terminals, filled, agree.to(torch.uint8), filled_sum)]
    dq_tot, dq_ff, stats = torch.empty(B * T, device=DEV), torch.empty(B * T, device=DEV), torch.empty(4, device=DEV)
    scratch = _lib.scratch(DEV) if scratch is None else scratch
    _lib.call("xb_wqmix_loss_fwd_bwd", *[_lib.ptr(x) for x in ins], B, n, T, mode, 0.1, 0.99, rows_total,
              _lib.ptr(dq_tot), _lib.ptr(dq_ff), _lib.ptr(stats), _lib.ptr(scratch))
    torch.cuda.synchronize()
    return dq_tot.cpu(), dq_ff.cpu(), stats.cpu()


SHAPES = [(1, 1, 1), (3, 60, 12), (5, 60, 9), (8, 1, 33), (16, 60, 2), (5, 1, 1)]   # (n, T, A)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("n,T,A", SHAPES)
@pytest.mark.parametrize("B", [1, 2, 31, 32, 33, 1024])
def test_kernels_match_float64(B, n, T, A, masked):
    if B == 1024 and T == 60 and n == 16:
        pytest.skip("covered by the smaller batches at this width")
    rng = np.random.default_rng(B * 1000 + n * 100 + T + A)
    ins = _select_inputs(rng, B, n, T, A, masked)
    for double_q in (True, False):
        want = R.select_ref(*ins, double_q)
        got = _run_select(*ins, double_q)
        for w, g, name in zip(want[:3], got[:3], ("q_eval_taken", "q_cent_taken", "q_next_cent")):
            assert torch.equal(g.double(), w), name                        # gathers times 0/1 masks: bit-exact
        assert torch.equal(got[3].long(), want[3]) and torch.equal(got[4].bool(), want[4])
        assert float(got[5]) == float(want[5])
    actions, agent_mask, filled = ins[4], ins[5], ins[6]
    greedy = want[3]
    # backward: both scatters, bit-exact (one product per element)
    from xuance_b200 import _lib
    de, dc = torch.randn(B * T, n), torch.randn(B * T, n)
    dq_all, dq_cent = torch.zeros(B, n, T + 1, A, device=DEV), torch.zeros(B, n, T + 1, A, device=DEV)
    # the device copies stay referenced until the kernel has run (a dropped temporary's block is reused at once)
    dev_in = [x.to(DEV) for x in (de, dc, actions, greedy.int(), agent_mask, filled)]
    _lib.call("xb_wqmix_select_bwd", *[_lib.ptr(x) for x in dev_in], B, n, T, A, _lib.ptr(dq_all), _lib.ptr(dq_cent))
    torch.cuda.synchronize()
    we, wc = R.select_bwd_ref(de, dc, actions, greedy, agent_mask, filled, A)
    assert torch.equal(dq_all.cpu().double(), we) and torch.equal(dq_cent.cpu().double(), wc)
    # loss
    rewards = torch.from_numpy(rng.normal(size=(B, n, T)).astype(np.float32))
    terminals = torch.from_numpy((rng.random((B, n, T)) < 0.2).astype(np.float32))
    q_tot, q_ff, q_ff_next = (torch.from_numpy(rng.normal(size=B * T).astype(np.float32)) for _ in range(3))
    fs = filled.sum().reshape(1)
    if float(fs) == 0:
        return
    for mode in (R.OW, R.CW):
        g_tot, g_ff, g_st = _run_loss(q_tot, q_ff, q_ff_next, rewards, terminals, filled, want[4], fs, mode, B * T)
        w_tot, w_ff, w_st = R.loss_ref(q_tot, q_ff, q_ff_next, rewards, terminals, filled, want[4], fs, mode, 0.1,
                                       0.99, B * T)
        scale = 1.0 / float(fs)
        np.testing.assert_allclose(g_tot.numpy(), w_tot.numpy(), rtol=1e-5, atol=1e-6 * scale)
        np.testing.assert_allclose(g_ff.numpy(), w_ff.numpy(), rtol=1e-5, atol=1e-6 * scale)
        np.testing.assert_allclose(g_st.numpy(), w_st.numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("G", [2, 3, 8])
def test_shards_sum_to_the_full_batch(G):
    rng = np.random.default_rng(G)
    B, n, T = 48, 5, 60
    rewards = torch.from_numpy(rng.normal(size=(B, n, T)).astype(np.float32))
    terminals = torch.from_numpy((rng.random((B, n, T)) < 0.2).astype(np.float32))
    filled = torch.from_numpy((rng.random((B, T)) < 0.8).astype(np.float32))
    agree = torch.from_numpy(rng.random(B * T) < 0.3)
    q_tot, q_ff, q_ff_next = (torch.from_numpy(rng.normal(size=B * T).astype(np.float32)) for _ in range(3))
    fs = filled.sum().reshape(1)
    for mode in (R.OW, R.CW):
        full = _run_loss(q_tot, q_ff, q_ff_next, rewards, terminals, filled, agree, fs, mode, B * T)
        parts = []
        for idx in np.array_split(np.arange(B), G):
            rows = torch.from_numpy((idx[:, None] * T + np.arange(T)[None]).reshape(-1))
            parts.append(_run_loss(q_tot[rows], q_ff[rows], q_ff_next[rows], rewards[idx], terminals[idx], filled[idx],
                                   agree[rows], fs, mode, B * T))
        assert torch.equal(torch.cat([p[0] for p in parts]), full[0])   # per-row gradients: identical arithmetic
        assert torch.equal(torch.cat([p[1] for p in parts]), full[1])
        np.testing.assert_allclose(sum(p[2].double() for p in parts).numpy(), full[2].numpy(), rtol=2e-6, atol=1e-7)


def test_launch_to_launch_bit_identity():
    rng = np.random.default_rng(5)
    ins = _select_inputs(rng, 1024, 5, 60, 12, True)
    a, b = _run_select(*ins, True), _run_select(*ins, True)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    rewards = torch.from_numpy(rng.normal(size=(1024, 5, 60)).astype(np.float32))
    terminals = torch.zeros(1024, 5, 60)
    q = [torch.from_numpy(rng.normal(size=1024 * 60).astype(np.float32)) for _ in range(3)]
    la = _run_loss(*q, rewards, terminals, ins[6], a[4], a[5], R.CW, 1024 * 60)
    lb = _run_loss(*q, rewards, terminals, ins[6], a[4], a[5], R.CW, 1024 * 60)
    assert all(torch.equal(x, y) for x, y in zip(la, lb))


# ---------------------------------------------------------------- the learner
def _product_model(n, obs_dim, A, S, hid, mix, hyper, ff):
    from xuance_b200.common import AgentGrouping, Discrete
    from xuance_b200.torch.rl_models import (Basic_RNN, AgentFeatureEncoder, DiscreteActionValueCritic, QMIX_Mixer,
                                             QMIX_FF_Mixer, WeightedMixingQNetwork)
    keys = [f"agent_{i}" for i in range(n)]
    rep = Basic_RNN(input_shape=(obs_dim,), hidden_sizes=None, initialize=nn.init.orthogonal_, activation=nn.ReLU,
                    device=DEV, fc_hidden_sizes=[hid], recurrent_hidden_size=hid, N_recurrent_layers=1, dropout=0,
                    rnn='GRU')
    q = nn.ModuleDict({'shared': DiscreteActionValueCritic(AgentFeatureEncoder(rep), Discrete(A), [hid], None,
                                                           nn.init.orthogonal_, nn.ReLU, DEV)})
    grouping = AgentGrouping.shared(keys)
    model = WeightedMixingQNetwork(grouping, q, QMIX_Mixer(S, mix, hyper, n, DEV), QMIX_FF_Mixer(S, ff, n, DEV),
                                   use_rnn=True, device=DEV).to(DEV)
    return keys, grouping, model


def _fixture_model():
    return _product_model(R.FIX_N, R.FIX_OBS, R.FIX_A, R.FIX_S, R.FIX_HID, R.FIX_MIX, R.FIX_HYPER, R.FIX_FF)


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _learner(grouping, model, **over):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import WQMIX_Learner
    cfg = dict(device=DEV, model_dir="/tmp/xb200_wqmix_models", use_cuda_graph=False)
    cfg.update(over)
    return WQMIX_Learner(Namespace(**cfg), grouping, model, BaseCallback())


@pytest.mark.parametrize("agent,double_q", R.FIX_CASES)
def test_learner_reproduces_the_reference_fixture(agent, double_q):
    """qmix_rnn_detach_q_eval=True: the reference as it runs (only the mixers train), across a target sync."""
    _no_tf32()
    d = np.load(GOLDEN)
    pre = f"{agent}/dq{int(double_q)}/"
    keys, grouping, model = _fixture_model()
    init = {k[len(pre) + 5:]: torch.from_numpy(d[k]) for k in d.files if k.startswith(pre + "init/")}
    model.load_state_dict(init, strict=True)                   # a reference state_dict loads strictly
    lrn = _learner(grouping, model, **R.fix_learner_config(agent, double_q), qmix_rnn_detach_q_eval=True)
    assert lrn.total_iters == int(d[pre + "total_iters"])
    for it in range(R.FIX_UPDATES):
        info = lrn.update(fixture_sample(d, pre, it, keys))
        got = [info[k] for k in R.FIX_INFO_KEYS]
        np.testing.assert_allclose(got, d[pre + "infos"][it], rtol=1e-4, atol=1e-6, err_msg=f"{pre}it{it}")
        if it in R.FIX_SNAPSHOTS:
            flat = np.concatenate([v.cpu().numpy().reshape(-1) for v in model.state_dict().values()])
            np.testing.assert_allclose(flat, d[f"{pre}after{it}"], rtol=1e-4, atol=2e-5, err_msg=f"{pre}after{it}")
    for k, v in model.state_dict().items():
        if k.startswith(("individual_q_networks", "individual_q_centralized")):
            assert torch.equal(v.cpu(), init[k]), k


def _intended_run(agent, double_q, graph, updates=4, seed=0):
    _no_tf32()
    torch.manual_seed(seed)
    n, obs_dim, A, S, T, B = 5, 72, 12, 98, 20, 8
    keys, grouping, model = _product_model(n, obs_dim, A, S, 64, 32, 64, 256)
    om = WQMIXModelOracle(n, obs_dim, A, S)
    model.load_state_dict(om.state_dict(), strict=True)
    cfg = R.fix_learner_config(agent, double_q)
    cfg.update(episode_length=T, use_grad_clip=True, grad_clip_norm=10.0)
    lrn = _learner(grouping, model, **cfg, qmix_rnn_detach_q_eval=False, use_cuda_graph=graph)
    orc = WQMIXLearnerOracle(om, keys, agent=agent, alpha=0.1, sync_frequency=2, double_q=double_q,
                             use_grad_clip=True, grad_clip_norm=10.0, end_factor_lr_decay=0.5,
                             total_iters=lrn.total_iters, detach_q_eval=False)
    rng = np.random.default_rng(seed + 1)
    infos = []
    for it in range(updates):
        s = R.fix_sample(rng, keys, B=B, T=T, obs_dim=obs_dim, A=A, S=S)
        ip, io = lrn.update(s), orc.update(s)
        infos.append((ip, io))
    return model, om, infos


@pytest.mark.parametrize("agent,double_q,graph", [("OWQMIX", True, False), ("CWQMIX", True, False),
                                                  ("CWQMIX", False, False), ("OWQMIX", True, True),
                                                  ("CWQMIX", True, True)])
def test_learner_matches_the_oracle_intended_computation(agent, double_q, graph):
    model, om, infos = _intended_run(agent, double_q, graph)
    for it, (ip, io) in enumerate(infos):
        for k in R.FIX_INFO_KEYS:
            np.testing.assert_allclose(ip[k], io[k], rtol=5e-4, atol=1e-5, err_msg=f"{k} it{it}")
    so, sp = om.state_dict(), model.state_dict()
    for k in so:
        np.testing.assert_allclose(sp[k].cpu().numpy(), so[k].numpy(), rtol=2e-3, atol=3e-4, err_msg=k)
    # the intended computation trains the central agent networks apart from the agent networks they were copied from
    w = "shared.critic_head.q_value.2.weight"
    assert not torch.equal(sp["individual_q_networks." + w], sp["individual_q_centralized." + w])


def test_graphed_update_is_bit_equal_to_eager():
    m_eager, _, i_eager = _intended_run("CWQMIX", True, False, updates=3, seed=4)
    m_graph, _, i_graph = _intended_run("CWQMIX", True, True, updates=3, seed=4)
    for (a, _), (b, _) in zip(i_eager, i_graph):
        assert a == b
    for (k, v), (_, w) in zip(m_eager.state_dict().items(), m_graph.state_dict().items()):
        assert torch.equal(v, w), k


def test_checkpoint_round_trip(tmp_path):
    _no_tf32()
    d = np.load(GOLDEN)
    pre = "CWQMIX/dq1/"
    cfg = dict(R.fix_learner_config("CWQMIX", True), end_factor_lr_decay=1.0)     # constant rate: the schedule is not saved
    keys, grouping, model = _fixture_model()
    lrn = _learner(grouping, model, **cfg)
    for it in range(2):
        lrn.update(fixture_sample(d, pre, it, keys))
    path = str(tmp_path / "wqmix.pth")
    lrn.save_model(path)
    keys2, grouping2, model2 = _fixture_model()
    lrn2 = _learner(grouping2, model2, **cfg)
    lrn2.load_model(path)
    for (k, v), (_, w) in zip(model.state_dict().items(), model2.state_dict().items()):
        assert torch.equal(v, w), k
    a, b = lrn.update(fixture_sample(d, pre, 2, keys)), lrn2.update(fixture_sample(d, pre, 2, keys))
    assert a == b


def _agent_config(**over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("wqmix", "sc2", "3m")
    base = dict(vectorize="Dummy_StarCraft2", parallels=8, buffer_size=64, batch_size=16, learning_rate=2e-3, gamma=0.5,
                start_greedy=1.0, end_greedy=0.05, decay_step_greedy=12000, start_training=200, running_steps=40000,
                n_epochs=4, sync_frequency=20, device=DEV, model_dir="/tmp/xb200_wqmix_models",
                log_dir="/tmp/xb200_wqmix_logs", episode_limit=20, p_death=0.02, distributed_training=False,
                use_cuda_graph=False, hidden_dim_hyper_net=32, hidden_dim_ff_mix_net=64)
    base.update(over)
    for k, v in base.items():
        setattr(cfg, k, v)
    return cfg


@pytest.mark.parametrize("agent", ["OWQMIX", "CWQMIX"])
def test_wqmix_learns_through_the_agent_registry(agent):
    """REGISTRY_Agents["OWQMIX"] / ["CWQMIX"] on the cue-following SMAC-shaped env (3m): the greedy team score rises."""
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.rl_models import WeightedMixingQNetwork
    cfg = _agent_config(agent=agent)
    envs = make_envs(cfg)
    ag = REGISTRY_Agents[agent](cfg, envs)
    assert isinstance(ag.model, WeightedMixingQNetwork) and ag.use_actions_mask
    before = float(np.mean(ag.test(16, make_envs(cfg))))
    info = ag.train(cfg.running_steps // cfg.parallels)
    assert {"loss_Qmix", "loss_central", "loss", "predictQ"} <= set(info) and np.isfinite(info["loss"])
    after = float(np.mean(ag.test(32, make_envs(cfg))))
    assert after > before + 2.0, (before, after)
    ag.finish()

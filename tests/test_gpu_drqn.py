"""GPU tests of DRQN: K13L (xb_lstm_seq_fwd / xb_lstm_seq_bwd) against the float64 restatement over sequence counts
around the 4-sequence slabs and past one wave, T from 1 to 200 and H from 1 to 128, zero and nonzero (h0, c0), with and
without (dhT, dcT); bit identity across launches and across subsets of S; the T = 1 acting step against step t of the
sequence kernel; the autograd Function against cuDNN nn.LSTM and under CUDA-graph capture; the replay, the learner and
seeded acting against the reference fixture; and a CartPole-v1 learning run of the shipped config."""
import os
import sys
from argparse import Namespace
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lstm_refs import lstm_fwd, lstm_bwd  # noqa: E402
from oracle_drqn import DRQNOracle  # noqa: E402
from oracle_drqn import seeded_state  # noqa: E402
from test_drqn import CASES, GOLDEN, initial_state, as_recorded, run_oracle, _model  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# K13's bound (test_gpu_gru_k13.py): the error relative to max(1, max|ref|), forward and backward.
TOL_FWD = 1e-6
TOL_BWD = 1e-6


def _lib():
    from xuance_b200 import _lib
    return _lib


def _problem(S, T, H, seed, nonzero_state=True, with_dT=True):
    """torch's default LSTM initialisation scale U(+-1/sqrt(H)) and unit-scale projected inputs."""
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / np.sqrt(H)
    u = lambda *shape: (torch.rand(*shape, generator=g, dtype=torch.float64) * 2 - 1) * k
    p = {"xg": torch.randn(S, T, 4 * H, generator=g, dtype=torch.float64), "w_hh": u(4 * H, H), "b_hh": u(4 * H),
         "h0": torch.randn(S, H, generator=g, dtype=torch.float64) * 0.5 if nonzero_state else None,
         "c0": torch.randn(S, H, generator=g, dtype=torch.float64) if nonzero_state else None,
         "dy": torch.randn(S, T, H, generator=g, dtype=torch.float64),
         "dhT": torch.randn(S, H, generator=g, dtype=torch.float64) if with_dT else None,
         "dcT": torch.randn(S, H, generator=g, dtype=torch.float64) if with_dT else None}
    return {k_: None if v is None else v.float() for k_, v in p.items()}


def _dev(t):
    return None if t is None else t.to(DEV).contiguous()


def k13l_fwd(xg, w_hh, b_hh, h0, c0, gates=True):
    L = _lib()
    S, T, G = xg.shape
    H = G // 4
    y = torch.empty(S, T, H, device=DEV)
    hT, cT = torch.empty(S, H, device=DEV), torch.empty(S, H, device=DEV)
    gt = torch.empty(S, T, 5 * H, device=DEV) if gates else None
    L.call("xb_lstm_seq_fwd", L.ptr(xg), L.ptr(w_hh), L.ptr(b_hh), L.ptr(h0), L.ptr(c0), S, T, H, L.ptr(y), L.ptr(hT),
           L.ptr(cT), L.ptr(gt))
    return y, hT, cT, gt


def k13l_bwd(dy, dhT, dcT, w_hh, gates, c0):
    L = _lib()
    S, T, H = dy.shape
    dxg = torch.empty(S, T, 4 * H, device=DEV)
    dh0, dc0 = torch.empty(S, H, device=DEV), torch.empty(S, H, device=DEV)
    L.call("xb_lstm_seq_bwd", L.ptr(dy), L.ptr(dhT), L.ptr(dcT), L.ptr(w_hh), L.ptr(gates), L.ptr(c0), S, T, H,
           L.ptr(dxg), L.ptr(dh0), L.ptr(dc0))
    return dxg, dh0, dc0


def _err(got, ref):
    ref = np.asarray(ref, np.float64)
    return float(np.abs(got.detach().cpu().double().numpy() - ref).max() / max(1.0, np.abs(ref).max()))


def _check(S, T, H, seed, nonzero_state, with_dT):
    p = _problem(S, T, H, seed, nonzero_state, with_dT)
    d = {k: _dev(v) for k, v in p.items()}
    y, hT, cT, gates = k13l_fwd(d["xg"], d["w_hh"], d["b_hh"], d["h0"], d["c0"])
    dxg, dh0, dc0 = k13l_bwd(d["dy"], d["dhT"], d["dcT"], d["w_hh"], gates, d["c0"])
    torch.cuda.synchronize()
    npy = lambda t: None if t is None else t.double().numpy()
    y_r, hT_r, cT_r, g_r = lstm_fwd(npy(p["xg"]), npy(p["w_hh"]), npy(p["b_hh"]), npy(p["h0"]), npy(p["c0"]))
    dxg_r, dh0_r, dc0_r = lstm_bwd(npy(p["dy"]), npy(p["dhT"]), npy(p["dcT"]), npy(p["w_hh"]), g_r, npy(p["c0"]))
    errs = {"y": _err(y, y_r), "hT": _err(hT, hT_r), "cT": _err(cT, cT_r), "gates": _err(gates, g_r)}
    errs_b = {"dxg": _err(dxg, dxg_r), "dh0": _err(dh0, dh0_r), "dc0": _err(dc0, dc0_r)}
    assert max(errs.values()) < TOL_FWD, errs
    assert max(errs_b.values()) < TOL_BWD, errs_b


@pytest.mark.parametrize("H", [1, 17, 32, 64, 100, 128])
@pytest.mark.parametrize("T", [1, 2, 50, 200])
@pytest.mark.parametrize("S", [1, 3, 4, 5, 8, 33, 640])
@pytest.mark.parametrize("nonzero_state,with_dT", [(False, False), (True, True)])
def test_k13l_matches_float64(S, T, H, nonzero_state, with_dT):
    _check(S, T, H, S * 7919 + T * 31 + H, nonzero_state, with_dT)


@pytest.mark.parametrize("nonzero_state,with_dT", [(False, True), (True, False)])
def test_k13l_matches_float64_mixed_states(nonzero_state, with_dT):
    _check(5, 50, 128, 3, nonzero_state, with_dT)
    _check(33, 2, 17, 4, nonzero_state, with_dT)


def test_k13l_beyond_one_wave_on_a_row_subset():
    S, T, H = 1 << 17, 2, 128
    p = _problem(S, T, H, 5)
    d = {k: _dev(v) for k, v in p.items()}
    y, hT, cT, gates = k13l_fwd(d["xg"], d["w_hh"], d["b_hh"], d["h0"], d["c0"])
    dxg, dh0, dc0 = k13l_bwd(d["dy"], d["dhT"], d["dcT"], d["w_hh"], gates, d["c0"])
    torch.cuda.synchronize()
    rows = np.r_[0:5, S // 2 - 3:S // 2 + 3, S - 5:S, np.random.default_rng(0).integers(0, S, 24)]
    npy = lambda t: t[rows].double().numpy()
    y_r, hT_r, cT_r, g_r = lstm_fwd(npy(p["xg"]), p["w_hh"].double().numpy(), p["b_hh"].double().numpy(),
                                    npy(p["h0"]), npy(p["c0"]))
    dxg_r, dh0_r, dc0_r = lstm_bwd(npy(p["dy"]), npy(p["dhT"]), npy(p["dcT"]), p["w_hh"].double().numpy(), g_r,
                                   npy(p["c0"]))
    ri = torch.as_tensor(rows, device=DEV)
    for got, ref, tol in ((y, y_r, TOL_FWD), (hT, hT_r, TOL_FWD), (cT, cT_r, TOL_FWD), (dxg, dxg_r, TOL_BWD),
                          (dh0, dh0_r, TOL_BWD), (dc0, dc0_r, TOL_BWD)):
        assert _err(got[ri], ref) < tol


def test_k13l_bit_identical_across_launches_and_subsets():
    S, T, H = 640, 20, 128
    p = _problem(S, T, H, 9)
    d = {k: _dev(v) for k, v in p.items()}
    a = k13l_fwd(d["xg"], d["w_hh"], d["b_hh"], d["h0"], d["c0"])
    b = k13l_fwd(d["xg"], d["w_hh"], d["b_hh"], d["h0"], d["c0"])
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    ga = k13l_bwd(d["dy"], d["dhT"], d["dcT"], d["w_hh"], a[3], d["c0"])
    gb = k13l_bwd(d["dy"], d["dhT"], d["dcT"], d["w_hh"], a[3], d["c0"])
    for u, v in zip(ga, gb):
        assert torch.equal(u, v)
    for idx in (torch.arange(3, 10), torch.tensor([639, 0, 17, 301, 5]), torch.arange(1, 640, 3)):
        idx = idx.to(DEV)
        sub = lambda t: None if t is None else t[idx].contiguous()
        fs = k13l_fwd(sub(d["xg"]), d["w_hh"], d["b_hh"], sub(d["h0"]), sub(d["c0"]))
        for u, v in zip(fs, a):
            assert torch.equal(u, v[idx])
        gs = k13l_bwd(sub(d["dy"]), sub(d["dhT"]), sub(d["dcT"]), d["w_hh"], fs[3], sub(d["c0"]))
        for u, v in zip(gs, ga):
            assert torch.equal(u, v[idx])


def test_acting_step_equals_sequence_step():
    S, T, H = 10, 12, 128
    p = _problem(S, T, H, 13)
    d = {k: _dev(v) for k, v in p.items()}
    y, hT, cT, gates = k13l_fwd(d["xg"], d["w_hh"], d["b_hh"], d["h0"], d["c0"])
    h, c = d["h0"], d["c0"]
    for t in range(T):
        yt, h, c, _ = k13l_fwd(d["xg"][:, t:t + 1].contiguous(), d["w_hh"], d["b_hh"], h, c, gates=False)
        assert torch.equal(yt[:, 0], y[:, t]) and torch.equal(c, gates[:, t, 4 * H:])
    assert torch.equal(h, hT) and torch.equal(c, cT)


def _lstm_pair(I, H, seed):
    torch.manual_seed(seed)
    ref = nn.LSTM(I, H, batch_first=True).to(DEV)
    mine = nn.LSTM(I, H, batch_first=True).to(DEV)
    mine.load_state_dict(ref.state_dict())
    return ref, mine


# cuDNN's LSTM sums in its own order (and may use other math for its GEMMs), so it is held to float32 round-off over a
# T-step recurrence rather than to the float64 bound above.
TOL_CUDNN = 2e-5


@pytest.mark.parametrize("S,T,H", [(8, 50, 128), (10, 1, 128), (5, 20, 17)])
def test_autograd_function_matches_cudnn_lstm(S, T, H):
    from xuance_b200.torch.rl_models import lstm_sequence
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    I = 24
    ref, mine = _lstm_pair(I, H, S + T + H)
    x = torch.randn(S, T, I, device=DEV)
    h0, c0 = torch.randn(S, H, device=DEV) * 0.5, torch.randn(S, H, device=DEV)
    xr, xm = x.clone().requires_grad_(), x.clone().requires_grad_()
    hr, hm = h0.clone().requires_grad_(), h0.clone().requires_grad_()
    cr, cm = c0.clone().requires_grad_(), c0.clone().requires_grad_()
    yr, (hTr, cTr) = ref(xr, (hr[None], cr[None]))
    ym, hTm, cTm = lstm_sequence(mine, xm, hm, cm)
    w = torch.randn_like(yr)
    ((yr * w).sum() + hTr.sum() + 0.5 * cTr.sum()).backward()
    ((ym * w).sum() + hTm.sum() + 0.5 * cTm.sum()).backward()
    close = lambda a, b: float((a - b).abs().max() / max(1.0, float(b.abs().max().detach())))
    assert close(ym, yr) < TOL_CUDNN and close(hTm, hTr[0]) < TOL_CUDNN and close(cTm, cTr[0]) < TOL_CUDNN
    for a, b in ((xm.grad, xr.grad), (hm.grad, hr.grad), (cm.grad, cr.grad)):
        assert close(a, b) < TOL_CUDNN
    for (n, pm), (_, pr) in zip(mine.named_parameters(), ref.named_parameters()):
        assert close(pm.grad, pr.grad) < TOL_CUDNN, n


def test_autograd_function_captures_in_a_cuda_graph():
    from xuance_b200.torch.rl_models import lstm_sequence
    S, T, I, H = 8, 50, 16, 128
    _, mine = _lstm_pair(I, H, 1)
    x = torch.randn(S, T, I, device=DEV)

    def step():
        for p in mine.parameters():
            p.grad = None
        y, hT, cT = lstm_sequence(mine, x)
        (y.square().sum() + cT.sum()).backward()
        return y.detach().clone(), [p.grad.clone() for p in mine.parameters()]

    y0, g0 = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], y0)
    for a, b in zip(out[1], g0):
        assert torch.equal(a, b)


# ---------------------------------------------------------------- replay against the reference fixture
def _replay_buffer():
    from xuance_b200.common import Box, Discrete, RecurrentOffPolicyBuffer
    return RecurrentOffPolicyBuffer(Box(-np.inf, np.inf, (3,)), Discrete(3), {}, 2, 12, 5, episode_length=20,
                                    lookup_length=8, device=DEV)


def _feed(buf, z):
    buf.begin(z["replay/init_obs"])
    for t in range(int(z["replay/n_steps"])):
        s = {k: z[f"replay/step{t}/{k}"] for k in ("next_obs", "actions", "rewards", "terminals", "done", "reset_obs")}
        buf.put(s["next_obs"], s["actions"], s["rewards"], s["terminals"])
        done = [e for e in range(2) if s["done"][e]]
        for e in done:
            buf.store(e)
        if done:
            buf.begin(s["reset_obs"], done)


def _check_samples(buf, z):
    for sd in (101, 102, 103):
        np.random.seed(sd)
        s = buf.sample()
        for k in ("obs", "actions", "rewards", "terminals"):
            ref = z[f"replay/sample{sd}/{k}"].astype(np.float32)
            got = s[k].cpu().numpy()
            assert got.shape == ref.shape and np.array_equal(got, ref), (sd, k)


def test_replay_matches_reference_and_round_trips():
    z = np.load(GOLDEN)
    buf = _replay_buffer()
    _feed(buf, z)
    assert buf.size == buf.n_size == 6
    order = [(buf.ptr - buf.size + p) % buf.n_size for p in range(buf.size)]
    assert np.array_equal(buf._len[order], z["replay/lengths"])
    _check_samples(buf, z)
    sd = buf.state_dict()
    fresh = _replay_buffer()
    fresh.load_state_dict(sd)
    _check_samples(fresh, z)


# ---------------------------------------------------------------- learner against the fixture and the oracle
def _learner(case, graph):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import DRQN_Learner
    name, rnn, H, obs_dim, rep_hidden, A, B, lookup, windows, clip, seed = case
    model = _model(rnn, H, obs_dim, rep_hidden, A).to(DEV)
    model.device = DEV
    model.representation.device = model.target_representation.device = DEV
    cfg = Namespace(learning_rate=1e-3, gamma=0.99, sync_frequency=2, use_grad_clip=clip, grad_clip_norm=0.5,
                    end_factor_lr_decay=0.5, running_steps=40, parallels=10, start_training=0, training_frequency=1,
                    device=DEV, use_cuda_graph=graph, model_dir="/tmp/xb_drqn_models")
    return model, DRQN_Learner(cfg, model, BaseCallback())


def _run(case, graph, z):
    name = case[0]
    model, learner = _learner(case, graph)
    template = {k: v.cpu() for k, v in model.state_dict().items()}
    model.load_state_dict({k: v.to(DEV) for k, v in initial_state(z, case, template).items()}, strict=True)
    infos = []
    for u in range(len(case[8])):
        s = {k: z[f"{name}/u{u}/{k}"] for k in ("obs", "actions", "rewards", "terminals")}
        s["batch_size"] = case[6]
        infos.append(learner.update(**s))
    return model, learner, infos


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_learner_matches_fixture_and_oracle_eager_and_graphed(case, tmp_path):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    z = np.load(GOLDEN)
    name = case[0]
    omodel, _, oinfos = run_oracle(z, case)
    m_e, l_e, i_e = _run(case, False, z)
    m_g, l_g, i_g = _run(case, True, z)
    for u in range(len(case[8])):
        for k in ("Qloss", "learning_rate", "predictQ"):
            ref = float(z[f"{name}/u{u}/info/{k}"])
            np.testing.assert_allclose(i_e[u][k], ref, rtol=1e-4, atol=1e-6, err_msg=f"{name} u{u} {k}")
            np.testing.assert_allclose(i_e[u][k], oinfos[u][k], rtol=1e-4, atol=1e-6)
            assert i_g[u][k] == i_e[u][k], (u, k)
    osd = omodel.state_dict()
    for k, v in m_e.state_dict().items():
        got = v.cpu().numpy()
        assert torch.equal(v, m_g.state_dict()[k]), k                       # graphed == eager, bit for bit
        np.testing.assert_allclose(got, osd[k].numpy(), rtol=1e-3, atol=2e-5, err_msg=k)
        ref = z[f"{name}/final/{k}"]
        np.testing.assert_allclose(as_recorded(name, got), ref, rtol=1e-3, atol=2e-4, err_msg=k)
    # checkpoint: save, load into a fresh learner, one more update each, same result
    path = str(tmp_path / "drqn.pth")
    l_e.save_model(path)
    m2, l2 = _learner(case, False)
    l2.load_model(path)
    for k, v in m_e.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k


# ---------------------------------------------------------------- agent
def _agent_config(**kw):
    cfg = dict(seed=1, device=DEV, parallels=4, buffer_size=400, batch_size=4, learning_rate=1e-3, gamma=0.99,
               start_greedy=0.5, end_greedy=0.01, decay_step_greedy=1000, sync_frequency=50, training_frequency=1,
               running_steps=1000, start_training=100, lookup_length=10, use_grad_clip=False, grad_clip_norm=0.5,
               representation="Basic_MLP", representation_hidden_size=[24], recurrent_hidden_size=17,
               recurrent_layer_N=1, dropout=0, rnn="LSTM", activation="relu", learner="DRQN_Learner",
               episode_length=50, env_name="Classic Control")
    cfg.update(kw)
    return SimpleNamespace(**cfg)


def test_seeded_acting_reproduces_reference_actions():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import DRQN_Agent
    z = np.load(GOLDEN)
    agent = DRQN_Agent(_agent_config(), observation_space=Box(-np.inf, np.inf, (5,)), action_space=Discrete(3))
    template = {k: v.cpu() for k, v in agent.model.state_dict().items()}
    agent.model.load_state_dict({k: v.to(DEV) for k, v in seeded_state(template, 21).items()}, strict=True)
    np.random.seed(21)
    states = agent.model.init_rnn_states(4)
    for t in range(6):
        out = agent.get_actions(z[f"act/step{t}/obs"], float(z[f"act/step{t}/egreedy"]), states)
        states = out.rnn_hidden
        assert np.array_equal(np.asarray(out.env_actions, np.int64), z[f"act/step{t}/actions"]), t
        np.testing.assert_allclose(states.hidden_states.cpu().numpy(), z[f"act/step{t}/h"], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(states.cell_states.cpu().numpy(), z[f"act/step{t}/c"], rtol=1e-5, atol=1e-6)


# CartPole-v1 with the shipped config, 60 000 environment steps (6 000 vector steps of 10 envs, ~5 900 updates).  On an
# H100 80GB HBM3 at 700 W this run scored a mean of 222.3 over 10 test episodes (125 to 314); the bound leaves headroom.
LEARN_STEPS = 60000
LEARN_MIN_SCORE = 120.0


def test_drqn_cartpole_learns():
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import DRQN_Agent
    cfg = get_arguments("drqn", "classic_control", "CartPole-v1",
                        parser_args=Namespace(device=DEV, running_steps=LEARN_STEPS, model_dir="/tmp/xb_models/drqn"))
    envs = make_envs(cfg)
    agent = DRQN_Agent(cfg, envs)
    assert agent.n_envs == 10 and agent.memory.n_size == 10000
    agent.train(LEARN_STEPS // agent.n_envs)
    assert {"Qloss", "learning_rate", "predictQ"} <= set(agent.logged)
    scores = agent.test(test_episodes=10)
    envs.close()
    agent.finish()
    print("DRQN CartPole-v1 test scores after %d steps:" % LEARN_STEPS, scores, "mean", np.mean(scores))
    assert np.mean(scores) > LEARN_MIN_SCORE, scores            # a random policy scores ~22

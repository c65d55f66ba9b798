"""GPU tests of SAC-Discrete: the K8D kernels against their float64 references at every A tier and row count (with the
probability edges, ties of min(q1, q2) and terminal rows), sharded minibatches, launch-to-launch determinism, the
out-of-range action rule, SACDIS_Learner against the torch-CPU oracle (auto alpha on / off, eager / graphed) and against the
reference fixture, K10 acting on a Discrete SAC agent, and CartPole-v1 learning through REGISTRY_Agents["SAC"]."""
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sacdis_refs import (sacdis_actor_ref, sacdis_critic_ref, edge_batch, probs_of, fixture_batch,  # noqa: E402
                         fixture_state_dict, OBS, A_FIX, HIDDEN)
from oracle_sacdis import SACDISModelOracle, SACDISLearnerOracle  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sacdis_update.npz")
BIG = 2048 * 256 + 3          # above the grid-stride threshold (2048 blocks of 256 rows)


def _lib():
    from xuance_b200 import _lib
    return _lib


def _run_actor(d, alpha, B_total=None, rows=None):
    L = _lib()
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    lg, q1, q2 = t(d["logits"]), t(d["q1"]), t(d["q2"])
    if rows is not None:
        lg, q1, q2 = lg[rows].contiguous(), q1[rows].contiguous(), q2[rows].contiguous()
    B, A = lg.shape
    dz = torch.empty_like(lg)
    stats = torch.full((4,), float("nan"), device=DEV)
    al = torch.tensor([alpha], device=DEV)
    L.call("xb_sacdis_actor_loss", L.ptr(lg), L.ptr(q1), L.ptr(q2), L.ptr(al), B, A, B_total or B, L.ptr(dz),
           L.ptr(stats), L.ptr(L.scratch(DEV)))
    return dz.cpu().numpy(), stats.cpu().numpy()


def _run_critic(d, alpha, gamma, B_total=None, rows=None):
    L = _lib()
    names = ("q1", "q2", "actions", "logits_next", "tq1", "tq2", "rew", "term")
    x = {k: torch.from_numpy(np.ascontiguousarray(d[k])).to(DEV) for k in names}
    if rows is not None:
        x = {k: v[rows].contiguous() for k, v in x.items()}
    B, A = x["q1"].shape
    dq1, dq2 = torch.full_like(x["q1"], float("nan")), torch.full_like(x["q2"], float("nan"))
    backup, stats = torch.empty_like(x["rew"]), torch.full((2,), float("nan"), device=DEV)
    al = torch.tensor([alpha], device=DEV)
    L.call("xb_sacdis_critic_loss", *[L.ptr(x[k]) for k in names], L.ptr(al), gamma, B, A, B_total or B, L.ptr(dq1),
           L.ptr(dq2), L.ptr(backup), L.ptr(stats), L.ptr(L.scratch(DEV)))
    return dq1.cpu().numpy(), dq2.cpu().numpy(), backup.cpu().numpy(), stats.cpu().numpy()


def _close(got, want, rtol, what):
    scale = max(float(np.abs(want).max()), 1e-30)
    np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol * scale, err_msg=what)


# every A tier (4 / 8 / 18 / 32 / 64, and A = 1) at 1, 255, 256, 257 rows; the grid-stride row count at one A per tier
CASES = [(A, B) for A in (1, 2, 4, 5, 8, 18, 32, 64) for B in (1, 255, 256, 257)] + [(A, BIG) for A in (3, 5, 18, 32, 64)]


@pytest.mark.parametrize("A,B", CASES)
def test_sacdis_kernels_tiers_and_row_counts(A, B):
    d = edge_batch(np.random.default_rng(A * 7 + B % 97), B, A)
    alpha, gamma = 0.37, 0.99
    dz, st = _run_actor(d, alpha)
    rz, rst = sacdis_actor_ref(d["logits"], d["q1"], d["q2"], alpha, B)
    _close(dz, rz, 2e-4, "dlogits")
    p = probs_of(d["logits"])
    assert np.all(dz[p == 0] == 0.0)
    np.testing.assert_allclose(st[:3], rst, rtol=2e-5, atol=1e-6)
    assert st[3] == 0.0
    dq1, dq2, bk, cst = _run_critic(d, alpha, gamma)
    r1, r2, rb, rq = sacdis_critic_ref(d["q1"], d["q2"], d["actions"], d["logits_next"], d["tq1"], d["tq2"], d["rew"],
                                       d["term"], alpha, gamma, B)
    np.testing.assert_allclose(bk, rb, rtol=1e-5, atol=1e-5)
    _close(dq1, r1, 1e-4, "dq1")
    _close(dq2, r2, 1e-4, "dq2")
    assert np.all(dq1[r1 == 0] == 0.0) and np.all(dq2[r2 == 0] == 0.0)
    np.testing.assert_allclose(cst[0], rq, rtol=2e-5)


@pytest.mark.parametrize("G", [2, 3, 8])
def test_sacdis_sharded_minibatch_sums_to_the_unsharded_launch(G):
    B, A = 257, 18
    d = edge_batch(np.random.default_rng(G), B, A)
    dz, st = _run_actor(d, 0.2)
    dq1, dq2, bk, cst = _run_critic(d, 0.2, 0.99)
    parts = np.array_split(np.arange(B), G)
    outs_a = [_run_actor(d, 0.2, B, torch.from_numpy(r).to(DEV)) for r in parts]
    outs_c = [_run_critic(d, 0.2, 0.99, B, torch.from_numpy(r).to(DEV)) for r in parts]
    np.testing.assert_array_equal(np.concatenate([o[0] for o in outs_a]), dz)
    np.testing.assert_array_equal(np.concatenate([o[0] for o in outs_c]), dq1)
    np.testing.assert_array_equal(np.concatenate([o[1] for o in outs_c]), dq2)
    np.testing.assert_array_equal(np.concatenate([o[2] for o in outs_c]), bk)
    np.testing.assert_allclose(sum(o[1] for o in outs_a)[:3], st[:3], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(sum(o[3][0] for o in outs_c), cst[0], rtol=1e-6)


def test_sacdis_statistics_are_bit_identical_from_launch_to_launch():
    d = edge_batch(np.random.default_rng(11), BIG, 5)
    a0, c0 = _run_actor(d, 0.2), _run_critic(d, 0.2, 0.99)
    for _ in range(2):
        a1, c1 = _run_actor(d, 0.2), _run_critic(d, 0.2, 0.99)
        assert a1[1].tobytes() == a0[1].tobytes() and c1[3].tobytes() == c0[3].tobytes()
        np.testing.assert_array_equal(a1[0], a0[0])


def test_out_of_range_actions_select_no_column():
    d = edge_batch(np.random.default_rng(3), 64, 4)
    d["actions"][:4] = [-1.0, 4.0, np.nan, 1e9]
    d["actions"][4] = 3.7                                    # truncates to 3, as act.long() does
    dq1, dq2, bk, st = _run_critic(d, 0.2, 0.99)
    assert np.all(dq1[:4] == 0) and np.all(dq2[:4] == 0) and np.isnan(st[0])
    assert dq1[4, 3] != 0 and np.count_nonzero(dq1[4]) == 1
    np.testing.assert_array_equal(np.isnan(bk), np.zeros(64, bool))


# ====================================================================================================== learner
def _product_model(obs_dim, A, rep_hidden, head_hidden):
    from copy import deepcopy
    from xuance_b200.common import Discrete
    from xuance_b200.torch.rl_models import (Basic_MLP, CategoricalActor, TwinDiscreteActionValueCritic,
                                             SoftActorCriticDiscrete)
    init, act = nn.init.orthogonal_, nn.ReLU
    rep = Basic_MLP((obs_dim,), list(rep_hidden), None, init, act, DEV)
    actor = CategoricalActor(rep, list(head_hidden), Discrete(A), None, init, act, DEV)
    critic = TwinDiscreteActionValueCritic(deepcopy(rep), Discrete(A), list(head_hidden), None, init, act, DEV)
    return SoftActorCriticDiscrete(actor, critic).to(DEV)


def _learner_cfg(auto, graph, **kw):
    cfg = dict(distributed_training=False, episode_length=1000, use_grad_clip=False, grad_clip_norm=0.5, device=DEV,
               model_dir="/tmp/xb", running_steps=100000, parallels=4, start_training=0, training_frequency=1,
               learning_rate_actor=1e-3, learning_rate_critic=1e-3, tau=0.005, gamma=0.99, alpha=0.2,
               use_automatic_entropy_tuning=auto, end_factor_lr_decay=0.7, use_cuda_graph=graph)
    cfg.update(kw)
    return Namespace(**cfg)


@pytest.mark.parametrize("auto,graph", [(False, False), (True, False), (False, True), (True, True)])
def test_sacdis_learner_matches_oracle(auto, graph):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import REGISTRY_Learners
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    obs_dim, A, B = 6, 7, 256
    om = SACDISModelOracle(obs_dim, A, (64,), (64,), (64,))
    model = _product_model(obs_dim, A, (64,), (64,))
    model.load_state_dict(om.state_dict(), strict=True)
    lrn = REGISTRY_Learners["SACDIS_Learner"](_learner_cfg(auto, graph, use_grad_clip=auto, grad_clip_norm=1.0), model,
                                              BaseCallback())
    orc = SACDISLearnerOracle(om, auto_alpha=auto, end_factor_lr_decay=0.7, total_iters=lrn.total_iters,
                              use_grad_clip=auto, grad_clip_norm=1.0)
    rng = np.random.default_rng(1)
    for it in range(5):
        s = {"obs": (rng.normal(size=(B, obs_dim)) * 3).astype(np.float32),
             "actions": rng.integers(0, A, B).astype(np.float32),
             "obs_next": (rng.normal(size=(B, obs_dim)) * 3).astype(np.float32),
             "rewards": rng.normal(size=B).astype(np.float32), "terminals": (rng.random(B) < 0.2).astype(np.float32)}
        io = orc.update(**s)
        ip = lrn.update(**{k: torch.from_numpy(v).to(DEV) for k, v in s.items()})
        for k in ("Qloss", "Ploss", "Qvalue"):
            np.testing.assert_allclose(ip[k], io[k], rtol=2e-4, atol=2e-5, err_msg=f"{k} it{it}")
        assert ip["actor_lr"] == io["actor_lr"] and ip["critic_lr"] == io["critic_lr"]
        if auto:
            np.testing.assert_allclose(ip["alpha"], io["alpha"], rtol=1e-5)
            np.testing.assert_allclose(ip["alpha_loss"], io["alpha_loss"], rtol=1e-3, atol=1e-6)
        else:
            assert "alpha" not in ip
    so, sp = om.state_dict(), model.state_dict()
    for k in so:
        np.testing.assert_allclose(sp[k].cpu().numpy(), so[k].numpy(), rtol=2e-3, atol=2e-4, err_msg=k)


@pytest.mark.parametrize("auto", [False, True])
def test_sacdis_learner_matches_reference_fixture(auto):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import REGISTRY_Learners
    torch.backends.cuda.matmul.allow_tf32 = False
    g = np.load(GOLDEN)
    pre = f"auto{int(auto)}/"
    model = _product_model(OBS, A_FIX, (HIDDEN,), (HIDDEN,))
    model.load_state_dict(fixture_state_dict(model.state_dict()), strict=True)
    lrn = REGISTRY_Learners["SACDIS_Learner"](_learner_cfg(auto, False), model, BaseCallback())
    assert lrn.total_iters == int(g[pre + "total_iters"])
    keys = ["Qloss", "Ploss", "Qvalue", "actor_lr", "critic_lr"] + (["alpha_loss", "alpha"] if auto else [])
    rng = np.random.default_rng(90 + auto)
    for it in range(3):
        s = fixture_batch(rng)
        info = lrn.update(**{k: torch.from_numpy(v).to(DEV) for k, v in s.items()})
        np.testing.assert_allclose([info[k] for k in keys], g[pre + "infos"][it], rtol=2e-4, atol=2e-5,
                                   err_msg=f"it{it}")
    for k, v in model.state_dict().items():
        np.testing.assert_allclose(v.cpu().numpy(), g[pre + "final/" + k], rtol=2e-3, atol=2e-4, err_msg=k)


# ====================================================================================================== acting
def _agent(A=5, **over):
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    cfg = get_arguments("sac", "classic_control", "CartPole-v1")
    for k, v in dict(device=DEV, model_dir="/tmp/xb_models/sacdis", logger=None, **over).items():
        setattr(cfg, k, v)
    return REGISTRY_Agents["SAC"](cfg, None, Box(-10, 10, (4,), np.float32), Discrete(A))


def test_discrete_sac_agent_acts_with_k10():
    from xuance_b200.torch.rl_models import SoftActorCriticDiscrete
    agent = _agent(A=5)
    assert isinstance(agent.model, SoftActorCriticDiscrete)
    assert type(agent.learner).__name__ == "SACDIS_Learner"
    obs = np.random.default_rng(0).normal(size=(10, 4)).astype(np.float32)
    with torch.no_grad():
        logits = agent.model.actor.logits(torch.from_numpy(obs).to(DEV)).cpu()
    greedy = agent.get_actions(obs, test_mode=True).env_actions
    np.testing.assert_array_equal(greedy, logits.argmax(-1).numpy())
    # stochastic: the empirical frequencies of one row repeated many times follow its probabilities
    big = np.repeat(obs[:1], 200000, axis=0)
    acts = agent.get_actions(big, test_mode=False).env_actions
    assert acts.dtype == np.int32 and acts.min() >= 0 and acts.max() < 5
    freq = np.bincount(acts, minlength=5) / acts.size
    p = torch.softmax(logits[0].double(), -1).numpy()
    np.testing.assert_allclose(freq, p, atol=5e-3)


# ====================================================================================================== learning
# CartPole-v1 with the shipped configs/sac/CartPole-v1.yaml (10 envs, B = 256, start_training 2000, one update per vector
# step), CARTPOLE_STEPS training steps.  Mean score of 10 greedy test episodes before -> after, on an H100 80GB HBM3 at its
# 700 W limit (a constant-action policy scores about 9-11):
#   seed 1: 9.4 -> 264.4   (the seed the test runs; 22 s including start-up)
#   seed 2: 11.5 -> 322.4
#   seed 3: 9.4 -> 251.6
# The required score, 125, is half the smallest.
CARTPOLE_STEPS = 30000
CARTPOLE_SCORE = 125.0


def test_sacdis_cartpole_learns():
    from xuance_b200 import get_runner
    runner = get_runner("sac", "classic_control", "CartPole-v1",
                        parser_args=Namespace(device=DEV, running_steps=CARTPOLE_STEPS,
                                              model_dir="/tmp/xb_models/sacdis_cartpole"))
    agent = runner.agent
    assert agent.n_envs == 10 and type(agent.learner).__name__ == "SACDIS_Learner"
    before = float(np.mean(agent.test(test_episodes=10)))
    runner.run("train", running_steps=CARTPOLE_STEPS)
    assert {"Qloss", "Ploss", "Qvalue", "actor_lr", "critic_lr"} <= set(agent.logged)
    after = float(np.mean(agent.test(test_episodes=10)))
    runner.finish()
    print("sacdis cartpole before %.1f after %.1f" % (before, after))
    assert after > CARTPOLE_SCORE and after > before, (before, after)

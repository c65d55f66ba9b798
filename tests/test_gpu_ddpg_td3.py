"""GPU tests of DDPG and TD3: the K8T kernels against the torch expressions (bit-exact) and their float64 references at
edge row counts and action widths, NaN propagation, in-place perturbation, sharded minibatches and launch-to-launch
determinism; DDPG_Learner / TD3_Learner against the torch-CPU oracle (delays 1-3, clip on / off, eager / graphed) and
against the reference fixture; checkpoints; exploration; and Pendulum-v1 learning through get_runner for both agents."""
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ddpg_refs import (critic_ref, actor_ref, perturb_ref, torch_exploration, torch_smoothing, torch_backup,  # noqa
                       loss_batch, action_batch, bounds, fixture_batch, fixture_state_dict, OBS, ACT, HIDDEN, LOW, HIGH,
                       SIGMA, NOISE_CLIP, DELAY, N_UPDATES, CLIP_NORM)
from oracle_ddpg import DDPGModelOracle, DDPGLearnerOracle  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ddpg_td3_update.npz")
BIG = 2048 * 256 + 3          # above the grid-stride threshold (2048 blocks of 256 threads)
KEYS = {"ddpg": ["Qloss", "Ploss", "Qvalue", "actor_lr", "critic_lr"],
        "td3": ["Qloss", "Ploss", "QvalueA", "QvalueB", "actor_lr", "critic_lr"]}


def _lib():
    from xuance_b200 import _lib
    return _lib


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _perturb(a, noise, scale, clip, low, high, out=None):
    L = _lib()
    a, noise, low, high = _t(a), _t(noise), _t(low), _t(high)
    out = torch.empty_like(a) if out is None else out
    L.call("xb_perturb_actions", L.ptr(a), L.ptr(noise), a.shape[0], a.shape[1], scale, clip, L.ptr(low), L.ptr(high),
           L.ptr(out))
    return out.cpu().numpy()


def _critic(d, twin, gamma, B_total=None, rows=None):
    L = _lib()
    x = {k: _t(d[k]) for k in ("q1", "q2", "tq1", "tq2", "rew", "term")}
    if rows is not None:
        x = {k: v[rows].contiguous() for k, v in x.items()}
    B = x["q1"].shape[0]
    q2, tq2 = (x["q2"], x["tq2"]) if twin else (None, None)
    dq1 = torch.full_like(x["q1"], float("nan"))
    dq2 = torch.full_like(x["q1"], float("nan")) if twin else None
    backup, stats = torch.empty_like(x["q1"]), torch.full((4,), float("nan"), device=DEV)
    L.call("xb_ddpg_critic_loss", L.ptr(x["q1"]), L.ptr(q2), L.ptr(x["tq1"]), L.ptr(tq2), L.ptr(x["rew"]),
           L.ptr(x["term"]), gamma, B, B_total or B, L.ptr(dq1), L.ptr(dq2), L.ptr(backup), L.ptr(stats),
           L.ptr(L.scratch(DEV)))
    c = lambda v: None if v is None else v.cpu().numpy()
    return c(dq1), c(dq2), c(backup), c(stats)


def _actor(d, twin, B_total=None, rows=None):
    L = _lib()
    q1, q2 = _t(d["q1"]), _t(d["q2"])
    if rows is not None:
        q1, q2 = q1[rows].contiguous(), q2[rows].contiguous()
    B = q1.shape[0]
    dq1 = torch.full_like(q1, float("nan"))
    dq2 = torch.full_like(q1, float("nan")) if twin else None
    stats = torch.full((4,), float("nan"), device=DEV)
    L.call("xb_ddpg_actor_loss", L.ptr(q1), L.ptr(q2 if twin else None), B, B_total or B, L.ptr(dq1), L.ptr(dq2),
           L.ptr(stats), L.ptr(L.scratch(DEV)))
    return dq1.cpu().numpy(), None if dq2 is None else dq2.cpu().numpy(), stats.cpu().numpy()


# ====================================================================================================== K8T-1
PERTURB_CASES = [(B, D) for B in (1, 255, 256, 257) for D in (1, 3, 6, 17, 64)] + [(BIG, 1), (BIG, 3), (BIG, 6)]


@pytest.mark.parametrize("B,D", PERTURB_CASES)
def test_perturb_is_the_torch_expression_bit_for_bit(B, D):
    rng = np.random.default_rng(B % 997 + D)
    low, high = bounds(D)
    a, n = action_batch(rng, B, D, low, high)
    tl, th = torch.from_numpy(low), torch.from_numpy(high)
    ta, tn = torch.from_numpy(a), torch.from_numpy(n)
    # exploration (no clip) and TD3 smoothing (clip), against the CPU and the CUDA evaluation of the torch expressions
    for scale, clip in ((0.3, -1.0), (SIGMA, NOISE_CLIP)):
        got = _perturb(a, n, scale, clip, low, high)
        if clip < 0:
            cpu = torch_exploration(ta, tn, scale, tl, th)
            gpu = torch_exploration(_t(a), _t(n), scale, _t(low), _t(high))
        else:
            cpu = torch_smoothing(ta, tn, scale, clip, tl, th)
            gpu = torch_smoothing(_t(a), _t(n), scale, clip, _t(low), _t(high))
        np.testing.assert_array_equal(got, cpu.numpy())
        np.testing.assert_array_equal(got, gpu.cpu().numpy())
        np.testing.assert_allclose(got, perturb_ref(a, n, np.float32(scale), np.float32(clip) if clip >= 0 else -1,
                                                    low, high), rtol=1e-6, atol=1e-6)
        if B * D >= 255:
            assert (got == low).any() and (got == high).any()      # both bounds bind
    if B >= 256:   # the clip binds: clipped noise strictly inside the bounds moves a by exactly +-clip
        got = _perturb(np.zeros_like(a), n, SIGMA, NOISE_CLIP, np.full(D, -9, np.float32), np.full(D, 9, np.float32))
        assert (got == np.float32(NOISE_CLIP)).any() and (got == -np.float32(NOISE_CLIP)).any()


def test_perturb_propagates_nan_and_works_in_place():
    rng = np.random.default_rng(4)
    B, D = 300, 6
    low, high = bounds(D)
    a, n = action_batch(rng, B, D, low, high)
    a[0, 0], n[1, 1], n[2, 2] = np.nan, np.nan, np.inf
    for scale, clip in ((0.3, -1.0), (SIGMA, NOISE_CLIP)):
        got = _perturb(a, n, scale, clip, low, high)
        assert np.isnan(got[0, 0]) and np.isnan(got[1, 1])
        assert got[2, 2] == (high[2] if clip < 0 else np.clip(a[2, 2] + np.float32(NOISE_CLIP), low[2], high[2]))
        f = torch_exploration if clip < 0 else (lambda x, y, s, lo, hi: torch_smoothing(x, y, s, clip, lo, hi))
        np.testing.assert_array_equal(got, f(torch.from_numpy(a), torch.from_numpy(n), scale, torch.from_numpy(low),
                                             torch.from_numpy(high)).numpy())
        # in place: out aliases a
        L = _lib()
        ta, tn, tl, th = _t(a), _t(n), _t(low), _t(high)
        L.call("xb_perturb_actions", L.ptr(ta), L.ptr(tn), B, D, scale, clip, L.ptr(tl), L.ptr(th), L.ptr(ta))
        np.testing.assert_array_equal(ta.cpu().numpy(), got)


# ====================================================================================================== K8T-2 / 3
LOSS_CASES = [(twin, B) for twin in (False, True) for B in (1, 255, 256, 257, BIG)]


@pytest.mark.parametrize("twin,B", LOSS_CASES)
def test_loss_kernels_row_counts(twin, B):
    d = loss_batch(np.random.default_rng(B % 991 + twin), B)
    gamma = 0.98
    dq1, dq2, bk, st = _critic(d, twin, gamma)
    r1, r2, rb, rst = critic_ref(d["q1"], d["q2"] if twin else None, d["tq1"], d["tq2"] if twin else None, d["rew"],
                                 d["term"], gamma, B)
    T = torch.from_numpy
    want = torch_backup(T(d["rew"]), T(d["term"]), gamma, T(d["tq1"]), T(d["tq2"]) if twin else None)
    np.testing.assert_array_equal(bk, want.numpy())                # the backup bit for bit
    np.testing.assert_allclose(bk, rb, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(dq1, r1, rtol=1e-5, atol=1e-5 * np.abs(r1).max())
    if twin:
        np.testing.assert_allclose(dq2, r2, rtol=1e-5, atol=1e-5 * np.abs(r2).max())
    np.testing.assert_allclose(st[:3], rst, rtol=2e-5, atol=1e-6)
    assert st[3] == 0.0 and (twin or st[2] == 0.0)
    a1, a2, ast = _actor(d, twin)
    s1, s2, pl = actor_ref(d["q1"], d["q2"] if twin else None, B)
    seed = np.float32(-1.0) / np.float32(B)
    np.testing.assert_array_equal(a1, np.full(B, seed * np.float32(0.5) if twin else seed, np.float32))
    if twin:
        np.testing.assert_array_equal(a2, a1)
    np.testing.assert_allclose(a1, s1, rtol=1e-6)
    np.testing.assert_allclose(ast[0], pl, rtol=2e-5, atol=1e-7)
    assert (ast[1:] == 0).all()


def test_actor_seeds_are_autograds_on_the_device():
    for twin in (False, True):
        d = loss_batch(np.random.default_rng(9), 257)
        a1, a2, _ = _actor(d, twin)
        q1, q2 = _t(d["q1"]).requires_grad_(True), _t(d["q2"]).requires_grad_(True)
        (-((q1 + q2) / 2.0).mean() if twin else -q1.mean()).backward()
        np.testing.assert_array_equal(a1, q1.grad.cpu().numpy())
        if twin:
            np.testing.assert_array_equal(a2, q2.grad.cpu().numpy())


@pytest.mark.parametrize("twin", [False, True])
def test_nan_target_propagates(twin):
    d = loss_batch(np.random.default_rng(2), 64, nan_rows=3)
    dq1, dq2, bk, st = _critic(d, twin, 0.99)
    assert np.isnan(bk[:3]).all() and np.isfinite(bk[3:]).all() and np.isnan(dq1[:3]).all() and np.isnan(st[0])
    if twin:   # torch.minimum: a NaN in either operand
        d = loss_batch(np.random.default_rng(2), 64)
        d["tq2"][5] = np.nan
        assert np.isnan(_critic(d, True, 0.99)[2][5])


@pytest.mark.parametrize("G", [2, 3, 8])
def test_sharded_minibatch_sums_to_the_unsharded_launch(G):
    B = 257
    d = loss_batch(np.random.default_rng(G), B)
    parts = np.array_split(np.arange(B), G)
    for twin in (False, True):
        full_c, full_a = _critic(d, twin, 0.98), _actor(d, twin)
        outs_c = [_critic(d, twin, 0.98, B, torch.from_numpy(r).to(DEV)) for r in parts]
        outs_a = [_actor(d, twin, B, torch.from_numpy(r).to(DEV)) for r in parts]
        for i in (0, 2) + ((1,) if twin else ()):
            np.testing.assert_array_equal(np.concatenate([o[i] for o in outs_c]), full_c[i])
        np.testing.assert_array_equal(np.concatenate([o[0] for o in outs_a]), full_a[0])
        np.testing.assert_allclose(sum(o[3] for o in outs_c)[:3], full_c[3][:3], rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(sum(o[2][0] for o in outs_a), full_a[2][0], rtol=1e-6, atol=1e-7)


def test_statistics_are_bit_identical_from_launch_to_launch():
    d = loss_batch(np.random.default_rng(11), BIG)
    for twin in (False, True):
        c0, a0 = _critic(d, twin, 0.98), _actor(d, twin)
        for _ in range(2):
            c1, a1 = _critic(d, twin, 0.98), _actor(d, twin)
            assert c1[3].tobytes() == c0[3].tobytes() and a1[2].tobytes() == a0[2].tobytes()
            np.testing.assert_array_equal(c1[0], c0[0])


# ====================================================================================================== learners
def _product_model(twin, obs_dim, act_dim, low, high, hidden, sigma=SIGMA, noise_clip=NOISE_CLIP):
    from copy import deepcopy
    from xuance_b200.common import Box
    from xuance_b200.torch.rl_models import (Basic_MLP, DeterministicActor, ActionValueCritic, TwinActionValueCritic,
                                             DeterministicActorCritic, TwinDelayedActorCritic)
    init, act = nn.init.orthogonal_, nn.ReLU
    space = Box(low, high, (act_dim,), np.float32)
    rep = Basic_MLP((obs_dim,), [hidden], None, init, act, DEV)
    actor = DeterministicActor(rep, [hidden], space, None, init, act, nn.Tanh, DEV)
    if twin:
        critic = TwinActionValueCritic(deepcopy(rep), space, [hidden], None, init, act, DEV)
        return TwinDelayedActorCritic(actor, critic, sigma, noise_clip).to(DEV)
    return DeterministicActorCritic(actor, ActionValueCritic(deepcopy(rep), space, [hidden], None, init, act, DEV)).to(DEV)


def _learner_cfg(graph, **kw):
    cfg = dict(distributed_training=False, episode_length=1000, use_grad_clip=False, grad_clip_norm=0.5, device=DEV,
               model_dir="/tmp/xb_ddpg", running_steps=64, parallels=4, start_training=0, training_frequency=1,
               learning_rate_actor=1e-3, learning_rate_critic=2e-3, tau=0.05, gamma=0.98, end_factor_lr_decay=0.5,
               actor_update_delay=DELAY, use_cuda_graph=graph)
    cfg.update(kw)
    return Namespace(**cfg)


def _learner(twin, model, cfg):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import REGISTRY_Learners
    return REGISTRY_Learners["TD3_Learner" if twin else "DDPG_Learner"](cfg, model, BaseCallback())


LEARNER_CASES = [("ddpg", 1, clip, graph) for clip in (False, True) for graph in (False, True)] + \
                [("td3", delay, clip, graph) for delay in (1, 2, 3) for clip in (False, True) for graph in (False, True)]


@pytest.mark.parametrize("algo,delay,clip,graph", LEARNER_CASES)
def test_learner_matches_oracle(algo, delay, clip, graph):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    twin = algo == "td3"
    obs_dim, act_dim, B, H = 6, 3, 256, 64
    low, high = np.array([-1, -0.5, -2], np.float32), np.array([1, 0.25, 2], np.float32)
    om = DDPGModelOracle(obs_dim, act_dim, low, high, twin, (H,), (H,), (H,), SIGMA, NOISE_CLIP)
    model = _product_model(twin, obs_dim, act_dim, low, high, H)
    model.load_state_dict(om.state_dict(), strict=True)
    lrn = _learner(twin, model, _learner_cfg(graph, use_grad_clip=clip, grad_clip_norm=0.3, actor_update_delay=delay))
    orc = DDPGLearnerOracle(om, lr_actor=1e-3, lr_critic=2e-3, tau=0.05, gamma=0.98, actor_update_delay=delay if twin else 1,
                            use_grad_clip=clip, grad_clip_norm=0.3, end_factor_lr_decay=0.5, total_iters=lrn.total_iters)
    rng = np.random.default_rng(1)
    n_actor = 0
    for it in range(7):
        s = {"obs": (rng.normal(size=(B, obs_dim)) * 3).astype(np.float32),
             "actions": rng.uniform(low, high, (B, act_dim)).astype(np.float32),
             "obs_next": (rng.normal(size=(B, obs_dim)) * 3).astype(np.float32),
             "rewards": rng.normal(size=B).astype(np.float32), "terminals": (rng.random(B) < 0.2).astype(np.float32)}
        noise = rng.normal(size=(B, act_dim)).astype(np.float32) * 1.5 if twin else None
        actor_step = (it + 1) % (delay if twin else 1) == 0
        n_actor += actor_step
        tgt = {k: v.flat.clone() for k, v in lrn._targets.items()}
        actor_before = lrn.optimizer['actor'].bucket.flat.clone()
        io = orc.update(noise_next=noise, **s)
        ip = lrn.update(noise_next=None if noise is None else _t(noise), **{k: _t(v) for k, v in s.items()})
        assert set(ip) == set(io), (set(ip), set(io))
        for k in io:
            if k.endswith("_lr"):
                assert ip[k] == io[k], k
            else:
                np.testing.assert_allclose(ip[k], io[k], rtol=2e-4, atol=2e-5, err_msg=f"{k} it{it}")
        if not actor_step:   # critic-only iteration: targets and actor bit-unchanged
            for k, v in lrn._targets.items():
                assert torch.equal(v.flat, tgt[k]), k
            assert torch.equal(lrn.optimizer['actor'].bucket.flat, actor_before)
        assert lrn.optimizer['actor'].step_count == n_actor and lrn.optimizer['critic'].step_count == it + 1
        st = [orc.opt_a.state[p].get("step", 0) for p in om.actor.parameters()]
        assert all(int(x) == n_actor for x in st)
    so, sp = om.state_dict(), model.state_dict()
    for k in so:
        np.testing.assert_allclose(sp[k].cpu().numpy(), so[k].numpy(), rtol=2e-3, atol=2e-4, err_msg=k)


@pytest.mark.parametrize("algo,clip", [("ddpg", False), ("ddpg", True), ("td3", False), ("td3", True)])
def test_learner_matches_reference_fixture(algo, clip):
    torch.backends.cuda.matmul.allow_tf32 = False
    g = np.load(GOLDEN)
    pre = f"{algo}/clip{int(clip)}/"
    twin = algo == "td3"
    model = _product_model(twin, OBS, ACT, LOW, HIGH, HIDDEN)
    model.load_state_dict(fixture_state_dict(model.state_dict()), strict=True)
    lrn = _learner(twin, model, _learner_cfg(False, use_grad_clip=clip, grad_clip_norm=CLIP_NORM))
    assert lrn.total_iters == int(g[pre + "total_iters"])
    rng = np.random.default_rng(70 + 2 * twin + clip)
    for it in range(N_UPDATES):
        s = fixture_batch(rng)
        noise = _t(g[pre + "noise"][it]) if twin else None
        info = lrn.update(noise_next=noise, **{k: _t(v) for k, v in s.items()})
        np.testing.assert_allclose([info.get(k, np.nan) for k in KEYS[algo]], g[pre + "infos"][it], rtol=2e-4,
                                   atol=2e-5, err_msg=f"it{it}")
        for k, v in model.state_dict().items():
            np.testing.assert_allclose(v.cpu().numpy(), g[f"{pre}it{it}/{k}"], rtol=2e-3, atol=2e-4,
                                       err_msg=f"it{it} {k}")


def test_reference_state_dict_loads_strictly_and_checkpoints_round_trip(tmp_path):
    g = np.load(GOLDEN)
    for algo in ("ddpg", "td3"):
        twin = algo == "td3"
        pre = f"{algo}/clip0/it3/"
        ref = {k[len(pre):]: torch.from_numpy(g[k]) for k in g if k.startswith(pre)}
        model = _product_model(twin, OBS, ACT, LOW, HIGH, HIDDEN)
        model.load_state_dict(ref, strict=True)
        lrn = _learner(twin, model, _learner_cfg(False))
        rng = np.random.default_rng(0)
        for _ in range(2):
            lrn.update(**{k: _t(v) for k, v in fixture_batch(rng).items()})
        path = str(tmp_path / f"{algo}.pth")
        lrn.save_model(path)
        model2 = _product_model(twin, OBS, ACT, LOW, HIGH, HIDDEN)
        lrn2 = _learner(twin, model2, _learner_cfg(False))
        lrn2.load_model(path)
        for k, v in model.state_dict().items():
            assert torch.equal(v, model2.state_dict()[k]), k
        for k in ("actor", "critic"):
            o1, o2 = lrn.optimizer[k], lrn2.optimizer[k]
            assert o1.step_count == o2.step_count and torch.equal(o1.exp_avg, o2.exp_avg)
        # the target buckets hold the loaded targets
        for k, mod in (("actor", model2.target_actor), ("critic", model2.target_critic)):
            assert lrn2._targets[k].flat.data_ptr() == next(mod.parameters()).data_ptr()


# ====================================================================================================== acting
def _agent(algo, **over):
    from xuance_b200.common import Box
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    cfg = get_arguments(algo, "classic_control", "Pendulum-v1")
    for k, v in dict(device=DEV, model_dir="/tmp/xb_models/" + algo, logger=None, **over).items():
        setattr(cfg, k, v)
    return REGISTRY_Agents[algo.upper()](cfg, None, Box(-8, 8, (3,), np.float32), Box(-2, 2, (1,), np.float32))


@pytest.mark.parametrize("algo", ["ddpg", "td3"])
def test_exploration_schedule_output_and_test_mode(algo):
    agent = _agent(algo)
    cfg = agent.config
    assert type(agent.learner).__name__ == algo.upper() + "_Learner"
    assert agent.delta_noise == (cfg.start_noise - cfg.end_noise) / (cfg.running_steps / agent.n_envs)
    for step in (0, 10, 250000, 499990, 500000):
        agent.current_step = step
        agent.noise_scale = cfg.start_noise
        agent._update_explore_factor()
        assert agent.noise_scale == cfg.start_noise - step * agent.delta_noise
    agent.noise_scale = 0.7
    obs = np.random.default_rng(0).normal(size=(10, 3)).astype(np.float32)
    n = torch.from_numpy(np.random.default_rng(1).normal(size=(10, 1)).astype(np.float32) * 3)
    with torch.no_grad():
        a = agent.model.act(_t(obs)).cpu()
    got = agent.get_actions(obs, noise=n.to(DEV)).env_actions
    want = torch_exploration(a, n, 0.7, torch.tensor([-2.0]), torch.tensor([2.0])).numpy()
    np.testing.assert_array_equal(got, want)
    assert (np.abs(got) == 2.0).any()
    np.testing.assert_array_equal(agent.get_actions(obs, test_mode=True).env_actions, a.numpy())
    torch.manual_seed(3)
    drawn = agent.get_actions(obs).env_actions                # the default draw is torch.randn_like on the device
    torch.manual_seed(3)
    np.testing.assert_array_equal(drawn, agent.exploration(agent.model.act(_t(obs)), None).cpu().numpy())


# ====================================================================================================== learning
# Pendulum-v1 with the shipped nested configs (10 envs, one update per vector step once start_training is reached) for
# PENDULUM[algo][0] training steps.  Mean score of 10 greedy test episodes before -> after, on an H100 80GB HBM3 at its 700 W
# limit (a random policy scores about -1200 to -1400; the tanh actor reaches only half of Pendulum's torque range, see
# DESIGN section 4):
#   DDPG,  60000 steps:  seed 1 -1279.2 -> -333.7 (the seed the test runs; 29 s),  seed 2 -1182.6 -> -503.6,
#                        seed 3 -1251.0 -> -297.3,  seed 4 -1226.3 -> -269.0,  seed 5 -1190.6 -> -294.8
#   TD3,  200000 steps:  seed 1 -1241.0 -> -293.9 (the seed the test runs; 64 s),  seed 2 -1262.9 -> -382.5,
#                        seed 3 -1285.2 -> -469.9,  seed 4 -1221.0 -> -411.8,  seed 5 -1406.8 -> -356.7
# TD3 updates its actor every third update at half DDPG's learning rate: at 60000 steps it had only reached -983 to -1090.
# The required score, -600, is below the worst run of either.
PENDULUM = {"ddpg": (60000, -600.0), "td3": (200000, -600.0)}   # (training steps, required mean test score)


@pytest.mark.parametrize("algo", ["ddpg", "td3"])
def test_pendulum_learns(algo):
    from xuance_b200 import get_runner
    steps, score = PENDULUM[algo]
    runner = get_runner(algo, "classic_control", "Pendulum-v1",
                        parser_args=Namespace(device=DEV, running_steps=steps, model_dir="/tmp/xb_models/%s_pendulum" % algo))
    agent = runner.agent
    assert agent.n_envs == 10 and type(agent.learner).__name__ == algo.upper() + "_Learner"
    before = float(np.mean(agent.test(test_episodes=10)))
    runner.run("train", running_steps=steps)
    assert {"Qloss", "Ploss", "actor_lr", "critic_lr"} <= set(agent.logged)
    after = float(np.mean(agent.test(test_episodes=10)))
    runner.finish()
    print("%s pendulum before %.1f after %.1f" % (algo, before, after))
    assert after > score and after > before, (before, after)

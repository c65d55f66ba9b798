"""CPU tests of the DDPG / TD3 stacks: the torch-CPU oracle against the reference fixture, the float64 kernel references
against torch autograd of the reference's expressions, the C-ABI argument checks (the mixed-NULL twin case included), the
nested configs and their lookup, the static config-key check over the new sources, and the out-of-scope errors."""
import ctypes
import os
import re
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ddpg_refs import (critic_ref, actor_ref, perturb_ref, torch_exploration, torch_smoothing, loss_batch,  # noqa
                       fixture_batch, fixture_state_dict, fixture_noise, OBS, ACT, HIDDEN, LOW, HIGH, SIGMA, NOISE_CLIP,
                       DELAY, N_UPDATES, CLIP_NORM)
from oracle_ddpg import DDPGModelOracle, DDPGLearnerOracle  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "ddpg_td3_update.npz")
KEYS = {"ddpg": ["Qloss", "Ploss", "Qvalue", "actor_lr", "critic_lr"],
        "td3": ["Qloss", "Ploss", "QvalueA", "QvalueB", "actor_lr", "critic_lr"]}


def _fixture_oracle(algo, clip, total_iters):
    twin = algo == "td3"
    m = DDPGModelOracle(OBS, ACT, LOW, HIGH, twin, (HIDDEN,), (HIDDEN,), (HIDDEN,), SIGMA, NOISE_CLIP)
    m.load_state_dict(fixture_state_dict(m.state_dict()))
    orc = DDPGLearnerOracle(m, lr_actor=1e-3, lr_critic=2e-3, tau=0.05, gamma=0.98, actor_update_delay=DELAY if twin else 1,
                            use_grad_clip=clip, grad_clip_norm=CLIP_NORM, end_factor_lr_decay=0.5, total_iters=total_iters)
    return m, orc


@pytest.mark.parametrize("algo,clip", [("ddpg", False), ("ddpg", True), ("td3", False), ("td3", True)])
def test_oracle_matches_reference_fixture(algo, clip):
    g = np.load(GOLDEN)
    pre = f"{algo}/clip{int(clip)}/"
    model, orc = _fixture_oracle(algo, clip, int(g[pre + "total_iters"]))
    assert sorted(model.state_dict()) == sorted(k[len(pre + "it0/"):] for k in g if k.startswith(pre + "it0/"))
    rng = np.random.default_rng(70 + 2 * (algo == "td3") + clip)
    for it in range(N_UPDATES):
        s = fixture_batch(rng)
        noise = g[pre + "noise"][it] if algo == "td3" else None
        info = orc.update(noise_next=noise, **s)
        want = g[pre + "infos"][it]
        got = [info.get(k, np.nan) for k in KEYS[algo]]
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-7, err_msg=f"it{it}")
        for k, v in model.state_dict().items():
            np.testing.assert_allclose(v.numpy(), g[f"{pre}it{it}/{k}"], rtol=1e-5, atol=1e-6, err_msg=f"it{it} {k}")


def test_fixture_reaches_the_clamps_and_the_delay():
    g = np.load(GOLDEN)
    for clip in (0, 1):
        inf = g[f"td3/clip{clip}/infos"]
        assert np.isnan(inf[0::2, 1]).all() and np.isfinite(inf[1::2, 1]).all()   # Ploss on actor iterations only
        n = g[f"td3/clip{clip}/noise"]
        assert (np.abs(n * np.float32(SIGMA)) > NOISE_CLIP).any()
        np.testing.assert_array_equal(n[0], fixture_noise(2000 + 10 * clip))
        # the actor's tanh alone leaves the middle component's bounds [-0.5, 0.25] (above 0.25)
        m = DDPGModelOracle(OBS, ACT, LOW, HIGH, True)
        m.load_state_dict({k[len(f"td3/clip{clip}/it0/"):]: torch.from_numpy(g[k]) for k in g
                           if k.startswith(f"td3/clip{clip}/it0/")})
        with torch.no_grad():
            a = m.act(torch.from_numpy(fixture_batch(np.random.default_rng(0))["obs"]))[:, 1]
        assert (a > HIGH[1]).any()
    # the delay: critic-only iterations leave the actor's learning rate where it was
    lr = g["td3/clip0/infos"][:, 4]
    assert lr[0] == 1e-3 and lr[1] < lr[0] and lr[2] == lr[1]


def test_reference_exploration_is_the_torch_expression():
    g = np.load(GOLDEN)
    a, n = torch.from_numpy(g["explore/actions"]), torch.from_numpy(g["explore/noise"])
    want = torch_exploration(a, n, float(g["explore/noise_scale"]), torch.from_numpy(LOW), torch.from_numpy(HIGH))
    np.testing.assert_array_equal(want.numpy(), g["explore/out"])
    assert (g["explore/out"] == LOW).any() and (g["explore/out"] == HIGH).any()


@pytest.mark.parametrize("twin", [False, True])
def test_float64_references_match_autograd(twin):
    rng = np.random.default_rng(3 + twin)
    B, gamma = 37, 0.97
    d = loss_batch(rng, B)
    t = lambda x: torch.tensor(x, dtype=torch.float64)
    q1, q2 = t(d["q1"]).requires_grad_(True), t(d["q2"]).requires_grad_(True)
    tq = torch.minimum(t(d["tq1"]), t(d["tq2"])) if twin else t(d["tq1"])
    y = t(d["rew"]) + gamma * (1 - t(d["term"])) * tq
    mse = torch.nn.functional.mse_loss
    loss = mse(q1, y) + (mse(q2, y) if twin else 0.0)
    loss.backward()
    d1, d2, bk, st = critic_ref(d["q1"], d["q2"] if twin else None, d["tq1"], d["tq2"] if twin else None, d["rew"],
                                d["term"], gamma, B)
    np.testing.assert_allclose(bk, y.numpy(), rtol=1e-14)
    np.testing.assert_allclose(d1, q1.grad.numpy(), rtol=1e-13, atol=1e-16)
    assert st[0] == pytest.approx(loss.item(), rel=1e-13) and st[1] == pytest.approx(q1.mean().item(), rel=1e-13)
    if twin:
        np.testing.assert_allclose(d2, q2.grad.numpy(), rtol=1e-13, atol=1e-16)
        assert st[2] == pytest.approx(q2.mean().item(), rel=1e-13)
    else:
        assert d2 is None and st[2] == 0.0
    a1, a2 = t(d["q1"]).requires_grad_(True), t(d["q2"]).requires_grad_(True)
    p = -((a1 + a2) / 2.0).mean() if twin else -a1.mean()
    p.backward()
    r1, r2, pl = actor_ref(d["q1"], d["q2"] if twin else None, B)
    np.testing.assert_array_equal(r1, a1.grad.numpy())
    assert pl == pytest.approx(p.item(), rel=1e-13)
    if twin:
        np.testing.assert_array_equal(r2, a2.grad.numpy())


def test_float32_seeds_are_autograds():
    """The kernels' float32 actor seeds, -(1/B) and (-(1/B))*0.5, are what float32 autograd writes."""
    for B in (1, 3, 100, 256, 257, 1000):
        q = torch.zeros(B, requires_grad=True)
        (-q.mean()).backward()
        assert q.grad[0].item() == np.float32(-1.0) / np.float32(B)
        a, b = torch.zeros(B, requires_grad=True), torch.zeros(B, requires_grad=True)
        (-((a + b) / 2.0).mean()).backward()
        assert a.grad[0].item() == (np.float32(-1.0) / np.float32(B)) * np.float32(0.5) == b.grad[0].item()


def test_perturb_reference_is_the_torch_expression_in_float64():
    rng = np.random.default_rng(8)
    low, high = np.array([-1, -0.5, -2.0]), np.array([1, 0.25, 2.0])
    a, n = rng.uniform(-3, 3, (50, 3)), rng.normal(0, 2, (50, 3))
    t = lambda x: torch.tensor(x, dtype=torch.float64)
    np.testing.assert_array_equal(perturb_ref(a, n, 0.3, -1, low, high),
                                  torch_exploration(t(a), t(n), 0.3, t(low), t(high)).numpy())
    np.testing.assert_array_equal(perturb_ref(a, n, 0.6, 0.5, low, high),
                                  torch_smoothing(t(a), t(n), 0.6, 0.5, t(low), t(high)).numpy())


def test_ddpg_entry_points_validate_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    j = ctypes.c_void_p(0x1000)
    EINVAL = -1
    for name in ("xb_perturb_actions", "xb_ddpg_critic_loss", "xb_ddpg_actor_loss"):
        assert name in _lib.exported_symbols() and hasattr(lib, name)

    def perturb(B=8, D=3, a=j, noise=j, low=j, high=j, out=j):
        return lib.xb_perturb_actions(a, noise, B, D, 0.1, -1.0, low, high, out, None)

    def critic(B=8, Bt=8, q1=j, q2=j, tq1=j, tq2=j, rew=j, term=j, dq1=j, dq2=j, backup=j, stats=j, scratch=j):
        return lib.xb_ddpg_critic_loss(q1, q2, tq1, tq2, rew, term, 0.99, B, Bt, dq1, dq2, backup, stats, scratch, None)

    def actor(B=8, Bt=8, q1=j, q2=j, dq1=j, dq2=j, stats=j, scratch=j):
        return lib.xb_ddpg_actor_loss(q1, q2, B, Bt, dq1, dq2, stats, scratch, None)
    assert perturb(B=0) == EINVAL and perturb(D=0) == EINVAL and perturb(D=-1) == EINVAL
    for k in ("a", "noise", "low", "high", "out"):
        assert perturb(**{k: None}) == EINVAL
    for f in (critic, actor):
        assert f(B=0) == EINVAL and f(Bt=4) == EINVAL and f(B=-1, Bt=-1) == EINVAL
        assert f(q1=None) == EINVAL and f(dq1=None) == EINVAL and f(stats=None) == EINVAL and f(scratch=None) == EINVAL
    for k in ("tq1", "rew", "term", "backup"):
        assert critic(**{k: None}) == EINVAL
    # the twin operands are all NULL (DDPG) or all set (TD3): any mix is refused
    for mix in (dict(q2=None), dict(tq2=None), dict(dq2=None), dict(q2=None, tq2=None), dict(tq2=None, dq2=None),
                dict(q2=None, dq2=None)):
        assert critic(**mix) == EINVAL, mix
    assert actor(q2=None) == EINVAL and actor(dq2=None) == EINVAL


def _cfg(algo, **over):
    from xuance_b200.common.common_tools import get_arguments
    d = dict(vars(get_arguments(algo, "classic_control", "Pendulum-v1")))
    d.update(device="cpu", **over)
    return Namespace(**d)


def test_configs_resolve_to_the_nested_files_with_the_reference_values():
    import yaml
    from xuance_b200.common import common_tools
    root = os.path.join(ROOT, "xuance_b200", "configs")
    for algo in ("ddpg", "td3"):
        nested = os.path.join(root, algo, "classic_control", "Pendulum-v1.yaml")
        assert os.path.exists(nested) and not os.path.exists(os.path.join(root, algo, "Pendulum-v1.yaml"))
        cfg = vars(common_tools.get_arguments(algo, "classic_control", "Pendulum-v1"))
        for k, v in yaml.safe_load(open(nested)).items():
            assert cfg[k] == v, (algo, k)
    d, t = _cfg("ddpg"), _cfg("td3")
    assert (d.agent, d.learner, d.representation, d.activation) == ("DDPG", "DDPG_Learner", "Basic_MLP", "relu")
    assert (d.representation_hidden_size, d.actor_hidden_size, d.critic_hidden_size) == ([256], [256], [256])
    assert (d.start_noise, d.end_noise, d.gamma, d.tau, d.batch_size, d.start_training) == (0.1, 0.1, 0.98, 0.005, 256,
                                                                                            1000)
    assert (t.agent, t.learner, t.representation, t.activation) == ("TD3", "TD3_Learner", "Basic_Identical", "leaky_relu")
    assert (t.actor_update_delay, t.start_noise, t.end_noise, t.training_frequency, t.start_training) == (3, 0.25, 0.05,
                                                                                                         2, 2000)
    assert (t.learning_rate_actor, t.learning_rate_critic, t.parallels, t.running_steps) == (0.0005, 0.001, 10, 500000)
    # the existing candidates keep their precedence
    assert common_tools.get_arguments("sac", "classic_control", "CartPole-v1").learner == "SACDIS_Learner"
    assert common_tools.get_arguments("ppo", "classic_control", "Pendulum-v1").agent == "PPO"
    with pytest.raises(AttributeError, match="mujoco"):
        common_tools.get_arguments("td3", "mujoco", "Ant-v4")


def test_nested_configs_define_every_key_their_classes_read():
    """The static check of test_host_logic over the two nested configs and the new sources: every ``config.X`` read without
    a getattr / hasattr default is a key of basic.yaml + the yaml."""
    import yaml
    root = os.path.join(ROOT, "xuance_b200")
    rd = lambda *p: open(os.path.join(root, *p)).read()
    base = set(yaml.safe_load(rd("configs", "basic.yaml")))
    src = "".join(rd(*f.split("/")) for f in ["torch/agents/off_policy.py", "torch/agents/ddpg_agent.py",
                                             "torch/learners/ddpg_learner.py", "torch/agents/agent.py",
                                             "torch/learners/learner.py"])
    hard = set(re.findall(r"(?<![a-zA-Z_])(?:self\.)?config\.([a-zA-Z_][a-zA-Z0-9_]*)\b(?!\s*=[^=])", src))
    soft = set(re.findall(r"(?:getattr|hasattr)\((?:self\.)?config,\s*.([a-zA-Z_0-9]+).", src))
    for algo in ("ddpg", "td3"):
        cfg = yaml.safe_load(open(os.path.join(root, "configs", algo, "classic_control", "Pendulum-v1.yaml")))
        assert not sorted(hard - soft - base - set(cfg)), algo
    # TD3's delay is read without a default: a TD3 config without it fails, as in the reference
    assert "actor_update_delay" in soft and 'getattr(config, "actor_update_delay")' in src


def test_registries():
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    assert {"DDPG", "TD3"} <= set(REGISTRY_Agents) and {"DDPG_Learner", "TD3_Learner"} <= set(REGISTRY_Learners)
    for name in ("MADDPG", "MATD3", "TD3BC", "TD3_BC"):
        assert name not in REGISTRY_Agents


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    obs = Box(-1, 1, (3,), np.float32)
    for algo, name in (("ddpg", "DDPG"), ("td3", "TD3")):
        with pytest.raises(ValueError, match="action_space must be Box"):
            REGISTRY_Agents[name](_cfg(algo), observation_space=obs, action_space=Discrete(3))
        with pytest.raises(NotImplementedError, match="one-dimensional"):
            REGISTRY_Agents[name](_cfg(algo), observation_space=obs, action_space=Box(-1, 1, (2, 3), np.float32))
        for env_name, what in (("MuJoCo", "MuJoCo"), ("Box2D", "Box2D"), ("Drones", "drone")):
            with pytest.raises(NotImplementedError, match=what):
                REGISTRY_Agents[name](_cfg(algo, env_name=env_name), observation_space=obs,
                                      action_space=Box(-1, 1, (1,), np.float32))
        with pytest.raises(NotImplementedError, match="device-side off-policy rollout"):
            REGISTRY_Agents[name](_cfg(algo, device_rollout=True), observation_space=obs,
                                  action_space=Box(-1, 1, (1,), np.float32))
    for algo in ("maddpg", "matd3", "td3bc"):
        with pytest.raises(AttributeError, match=algo):
            get_arguments(algo, "mpe", "simple_spread_v3")

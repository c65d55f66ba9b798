"""CPU tests of the C51 / QR-DQN stacks: the torch-CPU oracle against the reference fixture, the float64 kernel references
against torch autograd of the reference's expressions (Tz on an atom, clamping at both ends, ter = 1 rows, probabilities
that underflow to 0, A = 1, N = 2), the float32 scalar conventions the kernels follow, the C-ABI argument checks, the
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
from dist_refs import (greedy_ref, c51_ref, qrdqn_ref, torch_tz, torch_projection, torch_qr_backup,  # noqa: E402
                       torch_c51_loss, torch_qrdqn_loss, supports_of, loss_batch, fixture_batch, fixture_state_dict,
                       OBS, HIDDEN, N_ACT, ATOMS, QUANTILES, V_MIN, V_MAX, GAMMA, LR, SYNC, N_UPDATES, CLIP_NORM)
from oracle_dist import DistModelOracle, DistLearnerOracle  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "c51_qrdqn_update.npz")
N_OF = {"c51": ATOMS, "qrdqn": QUANTILES}


def _fixture_oracle(algo, clip, total_iters):
    m = DistModelOracle(algo, OBS, N_ACT, N_OF[algo], (HIDDEN,), (HIDDEN,), V_MIN, V_MAX)
    m.load_state_dict(fixture_state_dict(m.state_dict()))
    orc = DistLearnerOracle(m, lr=LR, gamma=GAMMA, sync_frequency=SYNC, use_grad_clip=clip, grad_clip_norm=CLIP_NORM,
                            end_factor_lr_decay=0.5, total_iters=total_iters)
    return m, orc


@pytest.mark.parametrize("algo,clip", [("c51", False), ("c51", True), ("qrdqn", False), ("qrdqn", True)])
def test_oracle_matches_reference_fixture(algo, clip):
    g = np.load(GOLDEN)
    pre = f"{algo}/clip{int(clip)}/"
    model, orc = _fixture_oracle(algo, clip, int(g[pre + "total_iters"]))
    assert sorted(model.state_dict()) == sorted(k[len(pre + "it0/"):] for k in g if k.startswith(pre + "it0/"))
    for k, v in model.state_dict().items():
        np.testing.assert_array_equal(v.numpy(), g[f"{pre}init/{k}"], err_msg=k)
    rng = np.random.default_rng(80 + 2 * (algo == "qrdqn") + clip)
    for it in range(N_UPDATES):
        info = orc.update(**fixture_batch(rng))
        np.testing.assert_allclose([info["Qloss"], info["learning_rate"]], g[pre + "infos"][it], rtol=1e-5, atol=1e-7,
                                   err_msg=f"it{it}")
        for k, v in model.state_dict().items():
            np.testing.assert_allclose(v.numpy(), g[f"{pre}it{it}/{k}"], rtol=1e-5, atol=1e-6, err_msg=f"it{it} {k}")


def test_fixture_crosses_a_target_sync_and_reaches_both_clamps():
    g = np.load(GOLDEN)
    for algo in ("c51", "qrdqn"):
        for clip in (0, 1):
            pre = f"{algo}/clip{clip}/"
            w = lambda it, net: g[f"{pre}it{it}/{net}.model.0.weight"]
            assert not np.array_equal(w(0, "eval_Z_head"), w(0, "target_Z_head"))       # the target lags ...
            np.testing.assert_array_equal(w(1, "eval_Z_head"), w(1, "target_Z_head"))   # ... until the copy at 2
            np.testing.assert_array_equal(w(3, "representation"), w(3, "target_representation"))
            assert not np.array_equal(w(2, "eval_Z_head"), w(2, "target_Z_head"))
    np.testing.assert_array_equal(g["c51/clip0/it3/supports"], supports_of(V_MIN, V_MAX, ATOMS).numpy())
    # the clip binds: the clipped run moves the weights less on the first update
    d = lambda c: np.abs(g[f"c51/clip{c}/it0/eval_Z_head.model.2.weight"] - g[f"c51/clip{c}/init/eval_Z_head.model.2.weight"])
    assert d(1).max() <= d(0).max()
    rng = np.random.default_rng(80)
    s = fixture_batch(rng)
    tz = torch_tz(torch.from_numpy(s["rewards"]), torch.from_numpy(s["terminals"]), supports_of(V_MIN, V_MAX, ATOMS),
                  GAMMA, V_MIN, V_MAX)
    assert (tz == V_MIN).any() and (tz == V_MAX).any() and (s["terminals"] == 1).any()


def _t64(x, grad=False):
    return torch.tensor(np.asarray(x), dtype=torch.float64, requires_grad=grad)


C51_CASES = [(37, 3, 51), (20, 1, 51), (25, 4, 2), (9, 18, 64), (33, 5, 33)]


@pytest.mark.parametrize("B,A,N", C51_CASES)
def test_c51_reference_matches_autograd(B, A, N):
    rng = np.random.default_rng(B * 100 + A + N)
    d = loss_batch(rng, B, A, N)
    sup = supports_of(-10.0, 10.0, N).double()
    ze = _t64(d["z_eval"], True)
    loss, ta = torch_c51_loss(ze, _t64(d["z_next"]), sup, torch.from_numpy(d["actions"]), _t64(d["rew"]),
                              _t64(d["ter"]), GAMMA, -10.0, 10.0, 20.0 / (N - 1))
    loss.backward()
    dl, rta, rl, tz, target = c51_ref(d["z_eval"], d["z_next"], sup.numpy(), d["actions"], d["rew"], d["ter"], GAMMA,
                                      -10.0, 10.0, B)
    np.testing.assert_array_equal(rta, ta.numpy())
    assert rl == pytest.approx(loss.item(), rel=1e-12)
    np.testing.assert_allclose(dl, ze.grad.numpy(), rtol=1e-10, atol=1e-15)
    # the regimes the batch is built to reach
    assert (tz == -10.0).any() and (tz == 10.0).any()
    assert tz[0, 0] == sup[1].item() and d["ter"][0] == 1.0          # Tz exactly on an atom: one weight of 1
    # the projection conserves probability (to the float32 spacing of the linspace supports)
    np.testing.assert_allclose(target.sum(-1), 1.0, rtol=1e-5)
    p = np.exp(d["z_eval"].astype(np.float64) - d["z_eval"].max(-1, keepdims=True))
    assert (p == 0).any() and (dl[p == 0] == 0).all()


@pytest.mark.parametrize("B,A,N", [(37, 3, 20), (20, 1, 20), (25, 4, 2), (9, 18, 64)])
def test_qrdqn_reference_matches_autograd(B, A, N):
    rng = np.random.default_rng(B * 10 + A + N)
    d = loss_batch(rng, B, A, N)
    ze = _t64(d["z_eval"], True)
    loss, ta = torch_qrdqn_loss(ze, _t64(d["z_next"]), torch.from_numpy(d["actions"]), _t64(d["rew"]), _t64(d["ter"]),
                                GAMMA)
    loss.backward()
    dq, rta, rl, y = qrdqn_ref(d["z_eval"], d["z_next"], d["actions"], d["rew"], d["ter"], GAMMA, B)
    np.testing.assert_array_equal(rta, ta.numpy())
    assert rl == pytest.approx(loss.item(), rel=1e-12)
    np.testing.assert_allclose(dq, ze.grad.numpy(), rtol=1e-12, atol=1e-16)
    np.testing.assert_array_equal(y[0], d["rew"][0])                  # ter = 1: the backup is the reward


def test_greedy_reference_is_the_models_expression():
    rng = np.random.default_rng(3)
    z = rng.normal(size=(50, 6, 51))
    z[:, 2] = z[:, 1]                                                  # ties pick the first index
    sup = supports_of(0, 200, 51).double()
    a, q, p = greedy_ref(z, sup.numpy())
    probs = torch.softmax(torch.from_numpy(z), -1)
    np.testing.assert_array_equal(a, (sup * probs).sum(-1).argmax(-1).numpy())
    np.testing.assert_allclose(p, probs.numpy(), rtol=1e-14)
    assert not (a == 2).any()
    a, q, _ = greedy_ref(z)
    np.testing.assert_array_equal(a, torch.from_numpy(z).mean(-1).argmax(-1).numpy())


def test_float32_scalar_conventions_of_the_kernels():
    """The float32 orders the K6Z kernels write with _rn intrinsics are torch 2.11's on the CPU: ``gamma * supports`` is a
    float32 product with float32(gamma); Tz is rew + (gamma*z)*(1 - ter), then the clamp; ``/ delta_z`` is a float32
    division by float32(delta_z) (not a product with the reciprocal); the QR backup is rew + (gamma*theta)*(1 - ter)."""
    rng = np.random.default_rng(5)
    f = np.float32
    B, N = 4000, 51
    recip_differs = []
    for v_min, v_max, gamma in ((-10, 10, 0.99), (0, 200, 0.99), (-3.5, 7.25, 0.97)):
        sup = supports_of(v_min, v_max, N)
        z = sup.numpy()
        rew = (rng.normal(size=B) * (v_max - v_min) * 0.4).astype(f)
        ter = (rng.random(B) < 0.3).astype(f)
        tz = torch_tz(torch.from_numpy(rew), torch.from_numpy(ter), sup, gamma, v_min, v_max).numpy()
        want = np.clip(rew[:, None] + (f(gamma) * z)[None, :] * (f(1) - ter[:, None]), f(v_min), f(v_max))
        np.testing.assert_array_equal(tz, want)
        dz = (v_max - v_min) / (N - 1)
        proj = torch_projection(torch.from_numpy(tz[:200]), sup, dz).numpy()
        want = np.clip(f(1) - np.abs(tz[:200, :, None] - z[None, None, :]) / f(dz), f(0), f(1))
        np.testing.assert_array_equal(proj, want)
        recip = np.clip(f(1) - np.abs(tz[:200, :, None] - z[None, None, :]) * f(1 / dz), f(0), f(1))
        recip_differs.append(not np.array_equal(proj, recip))
        th = rng.normal(size=(B, 20)).astype(f) * 5
        qr = torch_qr_backup(torch.from_numpy(rew), torch.from_numpy(ter), torch.from_numpy(th), gamma).numpy()
        np.testing.assert_array_equal(qr, rew[:, None] + (f(gamma) * th) * (f(1) - ter[:, None]))
    assert any(recip_differs)                       # the multiply-by-reciprocal form would not be torch's
    # the supports come from torch.linspace, which fills from both ends: not v_min + i*dz in float32
    lin = supports_of(-10, 10, 51).numpy()
    assert lin[0] == -10 and lin[-1] == 10 and lin.dtype == np.float32


def test_dist_entry_points_validate_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    j = ctypes.c_void_p(0x1000)
    EINVAL = -1
    for name in ("xb_dist_greedy", "xb_c51_loss_fwd_bwd", "xb_qrdqn_loss_fwd_bwd"):
        assert name in _lib.exported_symbols() and hasattr(lib, name)

    def greedy(B=8, A=4, N=51, z=j, sup=j, act=j, q=j, probs=j):
        return lib.xb_dist_greedy(z, sup, B, A, N, act, q, probs, None)

    def c51(B=8, A=4, N=51, Bt=8, ze=j, zn=j, sup=j, act=j, rew=j, ter=j, d=j, ta=j, td=j, stats=j, scratch=j):
        return lib.xb_c51_loss_fwd_bwd(ze, zn, sup, act, rew, ter, B, A, N, Bt, 0.99, -10.0, 10.0, 0.4, d, ta, td, stats,
                                       scratch, None)

    def qr(B=8, A=4, N=20, Bt=8, ze=j, zn=j, act=j, rew=j, ter=j, d=j, ta=j, stats=j, scratch=j):
        return lib.xb_qrdqn_loss_fwd_bwd(ze, zn, act, rew, ter, B, A, N, Bt, 0.99, d, ta, stats, scratch, None)
    for f in (greedy, c51, qr):
        assert f(B=0) == EINVAL and f(B=-1) == EINVAL
        assert f(N=1) == EINVAL and f(N=0) == EINVAL and f(N=65) == EINVAL       # N < 2 and over the 64 limit
        assert f(A=0) == EINVAL and f(A=257) == EINVAL                          # over the 256-action limit
    for f in (c51, qr):
        assert f(Bt=4) == EINVAL and f(B=-1, Bt=-1) == EINVAL
        for k in ("ze", "zn", "act", "rew", "ter", "d", "ta", "stats", "scratch"):
            assert f(**{k: None}) == EINVAL, (f.__name__, k)
    assert c51(sup=None) == EINVAL
    assert greedy(z=None) == EINVAL and greedy(act=None) == EINVAL
    assert greedy(sup=None) == EINVAL                # probabilities exist for C51 only


def _cfg(algo, env="classic_control", env_id="CartPole-v1", **over):
    from xuance_b200.common.common_tools import get_arguments
    d = dict(vars(get_arguments(algo, env, env_id)))
    d.update(device="cpu", **over)
    return Namespace(**d)


def test_configs_resolve_to_the_nested_files_with_the_reference_values():
    import yaml
    from xuance_b200.common import common_tools
    root = os.path.join(ROOT, "xuance_b200", "configs")
    for algo in ("c51", "qrdqn"):
        for env, env_id in (("classic_control", "CartPole-v1"), ("atari", "SyntheticAtari")):
            nested = os.path.join(root, algo, env, env_id + ".yaml")
            assert os.path.exists(nested) and not os.path.exists(os.path.join(root, algo, env_id + ".yaml"))
            assert not os.path.exists(os.path.join(root, algo, env + ".yaml"))
            cfg = vars(common_tools.get_arguments(algo, env, env_id))
            for k, v in yaml.safe_load(open(nested)).items():
                assert cfg[k] == v, (algo, k)
    c, q = _cfg("c51"), _cfg("qrdqn")
    assert (c.agent, c.learner, c.representation, c.atom_num, c.v_min, c.v_max) == ("C51DQN", "C51_Learner", "Basic_MLP",
                                                                                   51, 0, 200)
    assert (q.agent, q.learner, q.quantile_num, q.start_greedy, q.decay_step_greedy) == ("QRDQN", "QRDQN_Learner", 20,
                                                                                        0.25, 300000)
    assert (c.batch_size, c.sync_frequency, c.learning_rate, c.parallels) == (256, 100, 0.001, 10)
    ca, qa = _cfg("c51", "atari", "SyntheticAtari"), _cfg("qrdqn", "atari", "SyntheticAtari")
    for a in (ca, qa):
        assert (a.representation, a.filters, a.kernels, a.strides, a.q_hidden_size) == ("Basic_CNN", [32, 64, 64],
                                                                                         [8, 4, 3], [4, 2, 1], [512])
        assert (a.env_name, a.env_id, a.vectorize, a.batch_size, a.sync_frequency) == ("Atari", "SyntheticAtari",
                                                                                       "Dummy_Atari", 32, 500)
    # the out-of-scope simulators have no config
    for algo in ("c51", "qrdqn"):
        for env, env_id in (("box2d", "LunarLander-v3"), ("classic_control", "MountainCar-v0"),
                            ("classic_control", "Acrobot-v1")):
            with pytest.raises(AttributeError, match="no config"):
                common_tools.get_arguments(algo, env, env_id)


def test_nested_configs_define_every_key_their_classes_read():
    """The static check of test_host_logic over the four nested configs and the new sources: every ``config.X`` read
    without a getattr / hasattr default is a key of basic.yaml + the yaml."""
    import yaml
    root = os.path.join(ROOT, "xuance_b200")
    rd = lambda *p: open(os.path.join(root, *p)).read()
    base = set(yaml.safe_load(rd("configs", "basic.yaml")))
    src = "".join(rd(*f.split("/")) for f in ["torch/agents/off_policy.py", "torch/agents/dqn_agent.py",
                                             "torch/agents/dist_dqn_agent.py", "torch/learners/dqn_learner.py",
                                             "torch/learners/dist_dqn_learner.py",
                                             "torch/agents/agent.py", "torch/learners/learner.py"])
    hard = set(re.findall(r"(?<![a-zA-Z_])(?:self\.)?config\.([a-zA-Z_][a-zA-Z0-9_]*)\b(?!\s*=[^=])", src))
    soft = set(re.findall(r"(?:getattr|hasattr)\((?:self\.)?config,\s*.([a-zA-Z_0-9]+).", src))
    for algo in ("c51", "qrdqn"):
        for env, env_id in (("classic_control", "CartPole-v1"), ("atari", "SyntheticAtari")):
            cfg = yaml.safe_load(open(os.path.join(root, "configs", algo, env, env_id + ".yaml")))
            missing = hard - soft - base - set(cfg)
            # each algorithm's own head keys live only in its own configs
            missing -= {"quantile_num"} if algo == "c51" else {"atom_num", "v_min", "v_max"}
            missing -= {"PER_alpha", "PER_beta0"}         # PerDQN_Agent's, in the same module
            assert not sorted(missing), (algo, env)
    assert {"atom_num", "v_min", "v_max", "quantile_num"} <= hard


def test_registries():
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    assert REGISTRY_Agents["C51DQN"].__name__ == "C51_Agent" and REGISTRY_Agents["QRDQN"].__name__ == "QRDQN_Agent"
    assert {"C51_Learner", "QRDQN_Learner"} <= set(REGISTRY_Learners)
    for name in ("DRQN", "NoisyDQN"):
        assert name not in REGISTRY_Agents


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import REGISTRY_Agents
    obs = Box(-1, 1, (4,), np.float32)
    for algo, name in (("c51", "C51DQN"), ("qrdqn", "QRDQN")):
        with pytest.raises(ValueError, match="action_space must be Discrete"):
            REGISTRY_Agents[name](_cfg(algo), observation_space=obs, action_space=Box(-1, 1, (2,), np.float32))
        with pytest.raises(NotImplementedError, match="action masks"):
            REGISTRY_Agents[name](_cfg(algo, use_actions_mask=True), observation_space=obs, action_space=Discrete(2))
        key = "atom_num" if algo == "c51" else "quantile_num"
        for n in (1, 65):
            with pytest.raises(NotImplementedError, match="2 to 64 atoms"):
                REGISTRY_Agents[name](_cfg(algo, **{key: n}), observation_space=obs, action_space=Discrete(2))
        with pytest.raises(NotImplementedError, match="at most 256 actions"):
            REGISTRY_Agents[name](_cfg(algo), observation_space=obs, action_space=Discrete(257))

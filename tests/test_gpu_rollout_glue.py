"""GPU parity: device-side rollout glue (SURVEY.md section 8f-1) - K10 categorical act and K11 running mean/std +
observation normalise vs oracle/rollout.py and the reference outputs recorded in tests/golden/rollout_glue.npz, the
staged store path of the rollout buffer, and the PPO agent's ``device_rollout`` mode."""
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

from oracle.rollout import RunningMeanStdOracle, process_observation, categorical_act as act_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("N,A", [(300, 4), (256, 2), (64, 6), (1000, 18), (129, 19), (64, 32), (33, 40), (7, 64)])
def test_categorical_act_matches_oracle(N, A):
    from xuance_b200.torch.utils.rollout_glue import categorical_act
    rng = np.random.default_rng(N + A)
    logits = (rng.normal(size=(N, A)) * 2.5).astype(np.float32)
    u = rng.random(N).astype(np.float32)
    u[0] = 0.0
    lg = torch.from_numpy(logits).to(DEV)
    # --- inverse-CDF draw on supplied uniforms
    ai = torch.zeros(N, dtype=torch.int32, device=DEV)
    ent = torch.zeros(N, device=DEV)
    out = categorical_act(lg, uniforms=torch.from_numpy(u).to(DEV), actions_i32=ai, entropy=ent)
    a_o, logp_o, ent_o, cdf = act_oracle(logits, uniforms=u)
    a_p = out["actions"].cpu().numpy()
    assert np.array_equal(a_p, ai.cpu().numpy().astype(np.float32))
    # indices are exact wherever u is not within a few ulp of a CDF boundary (expf differs by <= 2 ulp between libm and CUDA)
    margin = np.abs(cdf - u[:, None]).min(axis=1)
    safe = margin > 2e-6
    assert safe.mean() > 0.99
    assert np.array_equal(a_p[safe].astype(np.int64), a_o[safe])
    # log-prob of the action the kernel chose, entropy
    logp_at = act_oracle(logits, forced_actions=a_p)[1]
    np.testing.assert_allclose(out["logp"].cpu().numpy(), logp_at, rtol=1e-5, atol=2e-6)
    np.testing.assert_allclose(ent.cpu().numpy(), ent_o, rtol=1e-5, atol=2e-6)
    # agrees with torch.distributions on the same logits (what the reference evaluates)
    d = torch.distributions.Categorical(logits=torch.from_numpy(logits))
    np.testing.assert_allclose(out["logp"].cpu().numpy(), d.log_prob(torch.from_numpy(a_p).long()).numpy(), rtol=1e-5,
                               atol=2e-6)
    # --- argmax mode
    out_d = categorical_act(lg)
    assert np.array_equal(out_d["actions"].cpu().numpy().astype(np.int64), act_oracle(logits)[0])
    # --- forced mode
    forced = rng.integers(0, A, N).astype(np.float32)
    out_f = categorical_act(lg, forced_actions=torch.from_numpy(forced).to(DEV))
    assert np.array_equal(out_f["actions"].cpu().numpy(), forced)
    np.testing.assert_allclose(out_f["logp"].cpu().numpy(), act_oracle(logits, forced_actions=forced)[1], rtol=1e-5,
                               atol=2e-6)


def test_categorical_act_distribution_and_edges():
    from xuance_b200.torch.utils.rollout_glue import categorical_act
    # empirical frequencies of the draw follow softmax(logits)
    logits = torch.tensor([[1.0, 0.0, -1.0, 2.0]], device=DEV).repeat(200000, 1)
    a = categorical_act(logits, uniforms=torch.rand(200000, device=DEV, generator=torch.Generator(DEV).manual_seed(0)))
    freq = torch.bincount(a["actions"].long(), minlength=4).double().cpu().numpy() / 200000
    np.testing.assert_allclose(freq, torch.softmax(logits[0].cpu().double(), 0).numpy(), atol=4e-3)
    # u just below 1 with a total mass that rounds below it: last action
    z = torch.zeros((1, 3), device=DEV)
    assert int(categorical_act(z, uniforms=torch.tensor([0.99999994], device=DEV))["actions"][0]) == 2
    # a dominant logit: probability-one action, log-prob 0, entropy 0
    z = torch.tensor([[0.0, 200.0, 0.0]], device=DEV)
    e = torch.zeros(1, device=DEV)
    o = categorical_act(z, uniforms=torch.tensor([0.5], device=DEV), entropy=e)
    assert int(o["actions"][0]) == 1 and float(o["logp"][0]) == 0.0 and float(e[0]) == 0.0


def test_categorical_and_rms_vs_reference_fixture():
    from xuance_b200.torch.utils.rollout_glue import categorical_act, DeviceRunningMeanStd
    g = np.load(os.path.join(G, "rollout_glue.npz"), allow_pickle=False)
    for A in (2, 4, 18):
        lg = torch.from_numpy(g[f"cat/{A}/logits"]).to(DEV)
        e = torch.zeros(lg.shape[0], device=DEV)
        o = categorical_act(lg, forced_actions=torch.from_numpy(g[f"cat/{A}/actions"]).to(DEV), entropy=e)
        np.testing.assert_allclose(o["logp"].cpu().numpy(), g[f"cat/{A}/log_prob"], rtol=1e-5, atol=2e-6)
        np.testing.assert_allclose(e.cpu().numpy(), g[f"cat/{A}/entropy"], rtol=1e-5, atol=2e-6)
        assert np.array_equal(categorical_act(lg)["actions"].cpu().numpy().astype(np.int64), g[f"cat/{A}/argmax"])
    for name, D in (("cartpole", 4), ("wide", 17)):
        rms = DeviceRunningMeanStd((D,), DEV)
        for it in range(6):
            x = torch.from_numpy(g[f"rms/{name}/x{it}"]).to(DEV)
            y = rms.update_and_normalize(x, 5)
            # float32 arithmetic in the reference's operation order (bit-identical when NumPy reduces row after row;
            # the asserted bound is a few float32 ulp of the accumulated sums)
            np.testing.assert_allclose(rms.mean.cpu().numpy(), g[f"rms/{name}/mean{it}"], rtol=2e-5, atol=1e-6)
            np.testing.assert_allclose(rms.var.cpu().numpy(), g[f"rms/{name}/var{it}"], rtol=2e-5, atol=1e-6)
            assert rms.count == float(g[f"rms/{name}/count{it}"])
            np.testing.assert_allclose(y.cpu().numpy(), g[f"rms/{name}/y{it}"], rtol=1e-4, atol=2e-5)


@pytest.mark.parametrize("N,shape", [(8, (4,)), (256, (17,)), (3, (5, 7)), (1, (130,))])
def test_device_running_mean_std_matches_oracle(N, shape):
    from xuance_b200.torch.utils.rollout_glue import DeviceRunningMeanStd
    rng = np.random.default_rng(N)
    rms, orc = DeviceRunningMeanStd(shape, DEV), RunningMeanStdOracle(shape)
    for it in range(5):
        x = (rng.normal(size=(N,) + shape) * (0.1 + 10 * it) - 3 * it).astype(np.float32)
        xd = torch.from_numpy(x).to(DEV)
        if it % 2 == 0:
            y = rms.update_and_normalize(xd, 5)
        else:
            rms.update(xd)
            y = rms.normalize(xd, 5)
        orc.update(x)
        np.testing.assert_allclose(rms.mean.cpu().numpy(), orc.mean, rtol=2e-5, atol=1e-6)
        np.testing.assert_allclose(rms.var.cpu().numpy(), orc.var, rtol=2e-5, atol=1e-6)
        assert rms.count == orc.count
        np.testing.assert_allclose(y.cpu().numpy(), process_observation(x, orc, 5), rtol=1e-4, atol=2e-5)
    st = rms.state()
    rms2 = DeviceRunningMeanStd(shape, DEV)
    rms2.load_state(st)
    assert torch.equal(rms2.mean, rms.mean) and torch.equal(rms2.var, rms.var) and rms2.count == rms.count


def test_store_staged_equals_store():
    """The staged path (policy outputs already on the device) leaves the same bytes in the buffer as ``store``."""
    from xuance_b200.common import DummyOnPolicyBuffer, DummyOnPolicyBuffer_Atari, Box, Discrete
    rng = np.random.default_rng(0)
    for atari, shape in ((False, (4,)), (True, (12, 12, 4))):
        cls = DummyOnPolicyBuffer_Atari if atari else DummyOnPolicyBuffer
        space = Box(0, 255, shape, np.uint8) if atari else Box(-10, 10, shape, np.float32)
        N, T = 6, 9
        a = cls(space, Discrete(4), {"old_logp": ()}, N, T, device=DEV)
        b = cls(space, Discrete(4), {"old_logp": ()}, N, T, device=DEV)
        slots = b.policy_slots()
        assert set(slots) == {"actions", "values", "aux:old_logp"}
        for t in range(T + 3):      # wraps the ring
            obs = rng.integers(0, 256, (N,) + shape, dtype=np.uint8) if atari else rng.normal(size=(N,) + shape).astype(np.float32)
            acts, vals = rng.integers(0, 4, N), rng.normal(size=N).astype(np.float32)
            logp, rews, terms = rng.normal(size=N).astype(np.float32), rng.normal(size=N).astype(np.float32), rng.random(N) < 0.3
            a.store(obs, acts, rews, vals, terms, {"old_logp": logp})
            slots["actions"].copy_(torch.from_numpy(acts.astype(np.float32)))
            slots["values"].copy_(torch.from_numpy(vals))
            slots["aux:old_logp"].copy_(torch.from_numpy(logp))
            b.store_staged(torch.from_numpy(obs).to(DEV), rews, terms)
            assert a.ptr == b.ptr and a.size == b.size
        assert torch.equal(a.observations, b.observations)
        assert torch.equal(a._fields[:a._n_store], b._fields[:b._n_store])


def test_ppo_cartpole_learns_with_device_rollout():
    from xuance_b200 import get_runner
    runner = get_runner("ppo", "classic_control", "CartPole-v1",
                        parser_args=Namespace(device="cuda:0", running_steps=40960, model_dir="/tmp/xb_models/ppo_dev",
                                              device_rollout=True))
    agent = runner.agent
    runner.run("train", running_steps=40960)
    assert {"actor_loss", "critic_loss", "entropy", "learning_rate", "predict_value", "clip_ratio"} <= set(agent.logged)
    if agent.use_obsnorm:       # host statistics were synchronised from the device copy
        assert agent.obs_rms.count > 40000 and np.all(np.isfinite(agent.obs_rms.mean))
    scores = agent.test(test_episodes=8)
    runner.finish()
    assert np.mean(scores) > 45.0, scores                  # a random policy scores ~22

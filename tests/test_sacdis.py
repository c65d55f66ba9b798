"""CPU tests of the SAC-Discrete stack: the torch-CPU oracle against the reference fixture, the float64 kernel references
against torch autograd of the reference's expressions (probabilities that underflow to exactly 0 or to subnormals, ties of
min(q1, q2), A = 1), the C-ABI argument checks, the config and the out-of-scope errors."""
import ctypes
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sacdis_refs import (sacdis_actor_ref, sacdis_critic_ref, edge_logits, edge_batch, probs_of, fixture_batch,  # noqa
                         fixture_state_dict, OBS, A_FIX, HIDDEN)
from oracle_sacdis import SACDISModelOracle, SACDISLearnerOracle  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sacdis_update.npz")
TINY32 = np.finfo(np.float32).tiny


def _fixture_model():
    m = SACDISModelOracle(OBS, A_FIX, (HIDDEN,), (HIDDEN,), (HIDDEN,))
    m.load_state_dict(fixture_state_dict(m.state_dict()))
    return m


@pytest.mark.parametrize("auto", [False, True])
def test_oracle_matches_reference_fixture(auto):
    g = np.load(GOLDEN)
    pre = f"auto{int(auto)}/"
    model = _fixture_model()
    assert sorted(model.state_dict()) == sorted(k[len(pre + "final/"):] for k in g if k.startswith(pre + "final/"))
    orc = SACDISLearnerOracle(model, auto_alpha=auto, end_factor_lr_decay=0.7, total_iters=int(g[pre + "total_iters"]))
    keys = ["Qloss", "Ploss", "Qvalue", "actor_lr", "critic_lr"] + (["alpha_loss", "alpha"] if auto else [])
    rng = np.random.default_rng(90 + auto)
    for it in range(3):
        s = fixture_batch(rng)
        if it == 0:
            with torch.no_grad():
                p, _, _, _ = model.Qpolicy(torch.from_numpy(s["obs"]))
            np.testing.assert_array_equal(p.numpy(), g[pre + "probs0"])
        info = orc.update(**s)
        np.testing.assert_allclose([info[k] for k in keys], g[pre + "infos"][it], rtol=1e-5, atol=1e-7)
    for k, v in model.state_dict().items():
        np.testing.assert_allclose(v.numpy(), g[pre + "final/" + k], rtol=1e-5, atol=1e-6, err_msg=k)


def test_fixture_reaches_the_probability_edges_and_records_the_reference_defect():
    g = np.load(GOLDEN)
    for a in (0, 1):
        p = g[f"auto{a}/probs0"]
        assert (p == 0).any() and ((p > 0) & (p < TINY32)).any()
    assert "action_space" in str(g["note/auto_alpha_error"])


def _autograd_actor(logits, q1, q2, alpha):
    """sacdis_learner.py:53-55 in float64 torch, the gradient to the logits by autograd."""
    z = torch.tensor(logits, dtype=torch.float64, requires_grad=True)
    p = torch.distributions.Categorical(logits=z).probs
    lp = torch.log(p + (p == 0.0).float() * 1e-8)
    mq = torch.min(torch.tensor(q1, dtype=torch.float64), torch.tensor(q2, dtype=torch.float64))
    loss = (p * (alpha * lp - mq)).sum(dim=1).mean()
    loss.backward()
    return z.grad.numpy(), np.array([loss.item(), mq.mean().item(), lp.mean().item()])


def _autograd_critic(q1, q2, actions, logits_next, tq1, tq2, rew, term, alpha, gamma):
    """sacdis_learner.py:63-70 in float64 torch."""
    t = lambda x: torch.tensor(np.asarray(x), dtype=torch.float64)
    a1, a2 = t(q1).requires_grad_(True), t(q2).requires_grad_(True)
    act = t(actions).unsqueeze(-1).long()
    p = torch.distributions.Categorical(logits=t(logits_next)).probs
    lp = torch.log(p + (p == 0.0).float() * 1e-8)
    target = (p * (torch.min(t(tq1), t(tq2)) - alpha * lp)).sum(dim=1).unsqueeze(-1)
    backup = t(rew).unsqueeze(-1) + (1 - t(term).reshape(-1, 1)) * gamma * target
    mse = torch.nn.functional.mse_loss
    loss = mse(a1.gather(1, act), backup.detach()) + mse(a2.gather(1, act), backup.detach())
    loss.backward()
    return a1.grad.numpy(), a2.grad.numpy(), backup.reshape(-1).detach().numpy(), loss.item()


def _float64_edges(z):
    """Rows whose float64 probabilities underflow to exactly 0 (a gap of 800) and to a subnormal (a gap of 720)."""
    z = z.astype(np.float64)
    if z.shape[1] >= 2:
        z[0, 1] = z[0].max() - 800.0
        z[1, 1] = z[1].max() - 720.0
        z[2, 0], z[2, 1] = 0.0, -800.0
        z[2, 2:] = -720.0
    return z


@pytest.mark.parametrize("A", [1, 2, 5, 18, 64])
def test_float64_references_match_autograd(A):
    rng = np.random.default_rng(A)
    B, alpha, gamma = 16, 0.37, 0.99
    d = edge_batch(rng, B, A)
    z, zn = _float64_edges(d["logits"]), _float64_edges(d["logits_next"])
    p = probs_of(z, torch.float64)
    if A >= 2:
        assert (p == 0).any() and ((p > 0) & (p < np.finfo(np.float64).tiny)).any()
    gz, st = _autograd_actor(z, d["q1"], d["q2"], alpha)
    dz, st2 = sacdis_actor_ref(z, d["q1"], d["q2"], alpha, B, torch.float64)
    np.testing.assert_allclose(dz, gz, rtol=1e-9, atol=1e-15)
    assert np.all(dz[p == 0] == 0.0) and np.all(gz[p == 0] == 0.0)
    np.testing.assert_allclose(st2, st, rtol=1e-10)
    g1, g2, bk, ql = _autograd_critic(d["q1"], d["q2"], d["actions"], zn, d["tq1"], d["tq2"], d["rew"], d["term"],
                                      alpha, gamma)
    d1, d2, bk2, ql2 = sacdis_critic_ref(d["q1"], d["q2"], d["actions"], zn, d["tq1"], d["tq2"], d["rew"], d["term"],
                                         alpha, gamma, B, torch.float64)
    np.testing.assert_allclose(bk2, bk, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(d1, g1, rtol=1e-10, atol=1e-15)
    np.testing.assert_allclose(d2, g2, rtol=1e-10, atol=1e-15)
    assert ql2 == pytest.approx(ql, rel=1e-12)


def test_edge_rows_reach_zero_and_subnormal_float32_probabilities():
    p = probs_of(edge_logits(np.random.default_rng(0), 8, 5))
    assert (p[0] == 0).sum() == 1 and ((p[1] > 0) & (p[1] < TINY32)).sum() == 1
    assert (p[2] == 0).sum() == 1 and ((p[2] > 0) & (p[2] < TINY32)).sum() == 1
    assert np.all(probs_of(edge_logits(np.random.default_rng(0), 8, 1)) == 1.0)   # A = 1: log_pi = 0, no gradient


def test_single_action_rows_have_no_policy_gradient():
    rng = np.random.default_rng(1)
    d = edge_batch(rng, 8, 1)
    dz, st = sacdis_actor_ref(d["logits"], d["q1"], d["q2"], 0.2, 8)
    assert np.all(dz == 0.0) and st[2] == 0.0
    np.testing.assert_allclose(st[0], -np.minimum(d["q1"], d["q2"]).astype(np.float64).mean(), rtol=1e-12)


def test_out_of_range_actions_select_no_column():
    rng = np.random.default_rng(2)
    d = edge_batch(rng, 6, 4)
    d["actions"][:3] = [-1.0, 4.0, np.nan]
    d1, d2, _, ql = sacdis_critic_ref(d["q1"], d["q2"], d["actions"], d["logits_next"], d["tq1"], d["tq2"], d["rew"],
                                      d["term"], 0.2, 0.99, 6)
    assert np.all(d1[:3] == 0) and np.all(d2[:3] == 0) and np.isnan(ql)
    assert np.count_nonzero(d1[3:]) == 3


def test_sacdis_entry_points_validate_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    j = ctypes.c_void_p(0x1000)
    EINVAL, ERANGE = -1, -3
    for name in ("xb_sacdis_actor_loss", "xb_sacdis_critic_loss"):
        assert name in _lib.exported_symbols() and hasattr(lib, name)

    def actor(B=8, A=5, Bt=8, logits=j, alpha=j, stats=j):
        return lib.xb_sacdis_actor_loss(logits, j, j, alpha, B, A, Bt, j, stats, j, None)

    def critic(B=8, A=5, Bt=8, actions=j, tq2=j, backup=j):
        return lib.xb_sacdis_critic_loss(j, j, actions, j, j, tq2, j, j, j, 0.99, B, A, Bt, j, j, backup, j, j, None)
    for f in (actor, critic):
        assert f(A=65) == ERANGE and f(A=0) == ERANGE
        assert f(B=0) == EINVAL and f(Bt=4) == EINVAL
    assert actor(logits=None) == EINVAL and actor(alpha=None) == EINVAL and actor(stats=None) == EINVAL
    assert critic(actions=None) == EINVAL and critic(tq2=None) == EINVAL and critic(backup=None) == EINVAL


def _cfg(**over):
    from xuance_b200.common.common_tools import get_arguments
    d = dict(vars(get_arguments("sac", "classic_control", "CartPole-v1")))
    d.update(over)
    return Namespace(**d)


def test_cartpole_config_carries_the_reference_hyper_parameters():
    cfg = _cfg()
    assert (cfg.agent, cfg.learner, cfg.policy, cfg.representation) == ("SAC", "SACDIS_Learner", "Categorical_SAC",
                                                                        "Basic_MLP")
    assert (cfg.batch_size, cfg.representation_hidden_size, cfg.actor_hidden_size, cfg.critic_hidden_size) == \
        (256, [128], [128], [128])
    assert (cfg.parallels, cfg.buffer_size, cfg.training_frequency, cfg.start_training) == (10, 200000, 2, 2000)
    assert (cfg.alpha, cfg.use_automatic_entropy_tuning, cfg.tau, cfg.gamma, cfg.activation) == (0.2, False, 0.005,
                                                                                                  0.99, "relu")
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    assert "SAC" in REGISTRY_Agents and "SACDIS_Learner" in REGISTRY_Learners


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import REGISTRY_Agents
    obs = Box(-1, 1, (4,), np.float32)
    with pytest.raises(NotImplementedError, match="64"):
        REGISTRY_Agents["SAC"](_cfg(), observation_space=obs, action_space=Discrete(65))
    with pytest.raises(NotImplementedError, match="use_actions_mask"):
        REGISTRY_Agents["SAC"](_cfg(use_actions_mask=True), observation_space=obs, action_space=Discrete(2))
    with pytest.raises(NotImplementedError, match="atari"):
        REGISTRY_Agents["SAC"](_cfg(env_name="Atari", representation="Basic_CNN"),
                               observation_space=Box(0, 255, (84, 84, 4), np.uint8), action_space=Discrete(6))

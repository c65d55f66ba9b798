"""CPU tests of the MAPPO stack: the float64 kernel references against torch autograd of the reference's formulas
(ties of torch.maximum / torch.min, clamp boundaries, Huber at |d| = delta, masked logits), the float32 ValueNorm
order against torch, the C-ABI argument checks, the config and the out-of-scope errors."""
import ctypes
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
MAPPO_CONFIG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "xuance_b200", "configs",
                            "mappo", "sc2", "5m_vs_6m.yaml")   # the reference's configs/mappo/sc2/ layout
from mappo_refs import mappo_loss_ref, value_norm_update_f32, finish_path_ref  # noqa: E402
from oracle_mappo import ValueNormOracle, MAPPOModelOracle, MAPPOLearnerOracle, MARLOnPolicyBufferOracle  # noqa: E402
from mappo_refs import mappo_buffer_steps, mappo_learner_batch  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mappo_update.npz")
KEYS = [f"agent_{i}" for i in range(3)]


def _autograd(logits, avail, actions, old_logp, adv, value, old_value, ret, mask, vn, clip, vclip, hdelta, vf, ent_c,
              R_total):
    """mappo_learner.py:55-126 in float64 torch, gradients by autograd."""
    t = lambda x: torch.tensor(np.asarray(x, np.float64))
    z = t(logits).requires_grad_(True)
    v = t(value).requires_grad_(True)
    zz = z.clone()
    if avail is not None:
        zz[t(avail) == 0] = -1e10
    dist = torch.distributions.Categorical(logits=zz)
    lp = dist.log_prob(t(actions).long())
    mk = t(mask)
    ratio = torch.exp(lp - t(old_logp))
    a = t(adv)
    s1, s2 = ratio * a, torch.clip(ratio, 1 - clip, 1 + clip) * a
    actor = -(torch.min(s1, s2) * mk).sum() / mk.sum()
    entropy = (dist.entropy() * mk).sum() / mk.sum()
    target = t(ret)
    if vn is not None:
        target = (target - vn[0]) / vn[1]
    L = nn.HuberLoss(reduction="none", delta=hdelta) if hdelta > 0 else (lambda x, y: (x - y) ** 2)
    if vclip > 0:
        vo = t(old_value)
        vc = vo + (v - vo).clamp(-vclip, vclip)
        lc = torch.max(L(v, target), L(vc, target))
    else:
        lc = L(v, target)
    critic = (lc * mk).sum() / mk.sum()
    loss = actor + vf * critic - ent_c * entropy
    loss.backward()
    stats = np.array([actor.item(), critic.item(), entropy.item(), v.sum().item() / R_total, loss.item()])
    return z.grad.numpy(), v.grad.numpy(), stats


def _inputs(rng, R, A, edge=False):
    logits = rng.normal(0, 1.5, (R, A))
    avail = (rng.random((R, A)) > 0.3).astype(np.uint8)
    actions = np.array([rng.choice(np.flatnonzero(r)) if r.any() else 0 for r in avail], np.float64)
    avail[np.arange(R), actions.astype(int)] = 1
    avail[0, :] = 0
    avail[0, int(actions[0])] = 1                 # a row with a single available action
    old_logp = rng.normal(-1.5, 0.5, R)
    adv = rng.normal(0, 1, R)
    value = rng.normal(0, 2, R)
    old_value = value + rng.normal(0, 0.1, R)
    ret = rng.normal(0, 15, R)
    mask = (rng.random(R) > 0.2).astype(np.float64)
    if edge:
        z = logits.copy()
        z[avail == 0] = -1e10
        lse = np.log(np.exp(z - z.max(1, keepdims=True)).sum(1)) + z.max(1)
        lp_a = z[np.arange(R), actions.astype(int)] - lse
        old_logp[:4] = lp_a[:4] - np.log([1.2, 0.8, 1.0, 1.2])   # ratio exactly-ish on the clip boundaries
        adv[4] = 0.0                                                # surrogate tie
        old_value[5:7] = value[5:7]                                 # value clip tie: both value losses equal
        ret[7], value[7] = 10.0, 0.0                                # Huber at |d| = delta
    return logits, avail, actions, old_logp, adv, value, old_value, ret, mask


@pytest.mark.parametrize("vclip,hdelta,use_vn,masked", [(0.2, 10.0, True, True), (0.0, 10.0, False, True),
                                                        (0.2, 0.0, True, False), (0.0, 0.0, False, False)])
def test_mappo_reference_matches_autograd(vclip, hdelta, use_vn, masked):
    rng = np.random.default_rng(3)
    R, A, clip = 64, 7, 0.2
    lg, av, act, olp, adv, v, vo, ret, mk = _inputs(rng, R, A, edge=True)
    av = av if masked else None
    vn = (0.5, 2.0) if use_vn else None
    if use_vn:
        ret[7] = 10.0 * 2.0 + 0.5
    gz, gv, st = _autograd(lg, av, act, olp, adv, v, vo, ret, mk, vn, clip, vclip, hdelta, 0.5, 0.01, R)
    dz, dv, st2 = mappo_loss_ref(lg, av, act, olp, adv, v, vo, ret, mk, vn, mk.sum(), R, clip, vclip, hdelta, 0.5,
                                 0.01)
    np.testing.assert_allclose(dz, gz, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(dv, gv, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(st2, st, rtol=1e-9, atol=1e-12)
    if masked:
        assert np.all(dz[av == 0] == 0.0)


def test_value_clip_tie_splits_the_gradient_in_halves():
    """torch.max of equal value losses: each side takes half; with v == v_old both sides carry the same gradient."""
    args = (np.zeros((1, 3)), None, np.zeros(1), np.zeros(1) - np.log(3), np.zeros(1), np.array([1.0]),
            np.array([1.0]), np.array([3.0]), np.ones(1))
    gz, gv, _ = _autograd(*args, None, 0.2, 0.1, 0.0, 1.0, 0.0, 1)
    _, dv, _ = mappo_loss_ref(*args, None, 1.0, 1, 0.2, 0.1, 0.0, 1.0, 0.0)
    assert gv[0] == pytest.approx(2 * (1.0 - 3.0)) and dv[0] == pytest.approx(gv[0])


def test_value_clip_symmetric_tie_takes_half_of_the_unclipped_gradient():
    """A tie of torch.maximum that tells the half split apart: |v - t| = |v_clipped - t| with the clipped branch blocked
    (v - v_old > c), so only the unclipped half passes: 0.5 * 2 * (v - t).  Exact in binary: v_old = 0, c = 0.25, v = 1,
    t = 0.625.  And the value-clip boundary v - v_old = c (inclusive: both halves pass, the full gradient)."""
    base = (np.zeros((1, 3)), None, np.zeros(1), np.zeros(1) - np.log(3), np.zeros(1))
    for v, ret, want in ((1.0, 0.625, 0.5 * 2 * 0.375), (0.25, 1.0, 2 * (0.25 - 1.0))):
        args = base + (np.array([v]), np.array([0.0]), np.array([ret]), np.ones(1))
        _, gv, _ = _autograd(*args, None, 0.2, 0.25, 0.0, 1.0, 0.0, 1)
        _, dv, _ = mappo_loss_ref(*args, None, 1.0, 1, 0.2, 0.25, 0.0, 1.0, 0.0)
        assert gv[0] == want and dv[0] == want


def test_ratio_on_the_clip_boundary_passes_the_gradient():
    """clip_range 0 puts ratio = 1 on both clamp boundaries (inclusive: the clipped surrogate's half passes too)."""
    args = (np.zeros((1, 2)), None, np.zeros(1), np.array([-np.log(2.0)]), np.array([1.0]), np.zeros(1), np.zeros(1),
            np.zeros(1), np.ones(1))
    gz, _, _ = _autograd(*args, None, 0.0, 0.0, 0.0, 1.0, 0.0, 1)
    dz, _, _ = mappo_loss_ref(*args, None, 1.0, 1, 0.0, 0.0, 0.0, 1.0, 0.0)
    np.testing.assert_allclose(dz, gz, rtol=1e-12)
    assert gz[0, 0] == pytest.approx(-0.5)       # d(-ratio)/dz_a = -(1 - p_a) in full, not half of it


def _vn_tuple(vn):
    m, var = vn.running_mean_var()
    return np.float32(m.item()), np.float32(np.sqrt(np.float32(var.item())))


@pytest.mark.parametrize("case", ["gae1_vn0", "gae1_vn1", "gae0_vn0"])
def test_buffer_oracle_matches_reference_fixture(case):
    g = np.load(GOLDEN)
    use_gae, use_vn = case == "gae1_vn0" or case == "gae1_vn1", case.endswith("vn1")
    rng = np.random.default_rng(5 + 2 * use_gae + use_vn)
    n_envs, T = 2, 12
    vn = None
    if use_vn:
        vn = ValueNormOracle()
        vn.update(torch.from_numpy(rng.normal(1.0, 4.0, (40, 1)).astype(np.float32)))
    steps, nexts, vn_upd = mappo_buffer_steps(rng, KEYS, n_envs, T, 12, 7)
    orc = MARLOnPolicyBufferOracle(3, n_envs, T, use_gae, 0.99, 0.95)
    for t, st in enumerate(steps):
        orc.store(KEYS, st)
        if t == 4:
            orc.finish_path(0, KEYS, {k: 0.0 for k in KEYS}, _vn_tuple(vn) if vn else None)
            if vn:
                vn.update(torch.from_numpy(vn_upd.reshape(-1, 1)))
    for e in range(n_envs):
        orc.finish_path(e, KEYS, nexts[e], _vn_tuple(vn) if vn else None)
    np.testing.assert_array_equal(orc.returns, g[f"buffer/{case}/returns"])
    np.testing.assert_array_equal(orc.advantages, g[f"buffer/{case}/advantages"])
    idx = g[f"buffer/{case}/idx"]
    np.testing.assert_allclose(orc.sample_advantages(idx), g[f"buffer/{case}/sample_advantages"], rtol=1e-5, atol=1e-6)


def _fixture_cfg():
    return Namespace(learning_rate=7e-4, clip_range=0.05, use_value_clip=True, value_clip_range=0.05,
                     use_value_norm=True, use_huber_loss=True, huber_delta=1.0, vf_coef=1.0, ent_coef=0.01,
                     use_grad_clip=True, grad_clip_norm=10.0)


def _fixture_init(model):
    from helpers import seeded_state_dict
    model.load_state_dict(seeded_state_dict(model.state_dict(), 31))
    return model


def test_learner_oracle_matches_reference_fixture():
    g = np.load(GOLDEN)
    model = _fixture_init(MAPPOModelOracle(12, 7))
    assert sorted(model.state_dict()) == sorted(k[len("learner/final/"):] for k in g if k.startswith("learner/final/"))
    orc = MAPPOLearnerOracle(model, _fixture_cfg())
    rng = np.random.default_rng(77)
    for it in range(3):
        b = mappo_learner_batch(rng, it, 32, KEYS, 12, 7)
        t = {k: torch.from_numpy(np.asarray(v).reshape(96, *np.asarray(v).shape[2:])) for k, v in b.items()
             if k != 'batch_size'}
        info = orc.update(t['obs'], t['actions'], t['log_pi_old'], t['advantages'], t['values'], t['returns'],
                          t['agent_mask'].float(), t['avail_actions'])
        got = [info[k] for k in ("actor_loss", "critic_loss", "entropy", "predict_value", "loss", "gradient_norm")]
        np.testing.assert_allclose(got, g["learner/infos"][it, :6], rtol=2e-6, atol=1e-7)
        np.testing.assert_allclose([orc.vn.running_mean.item(), orc.vn.running_mean_sq.item(),
                                    orc.vn.debiasing_term.item()], g[f"learner/vn_state/{it}"], rtol=1e-6)
    for k, v in model.state_dict().items():
        np.testing.assert_allclose(v.numpy(), g[f"learner/final/{k}"], rtol=1e-5, atol=1e-6, err_msg=k)


def test_fixture_reaches_the_clip_and_huber_regimes():
    """Update 1 of the fixture has every ratio outside the clip range; the normalised residuals straddle delta = 1."""
    g = np.load(GOLDEN)
    model = _fixture_init(MAPPOModelOracle(12, 7))
    orc = MAPPOLearnerOracle(model, _fixture_cfg())
    rng = np.random.default_rng(77)
    for it in range(2):
        b = mappo_learner_batch(rng, it, 32, KEYS, 12, 7)
        t = {k: torch.from_numpy(np.asarray(v).reshape(96, *np.asarray(v).shape[2:])) for k, v in b.items()
             if k != 'batch_size'}
        with torch.no_grad():
            z = model.logits(t['obs']).masked_fill(t['avail_actions'] == 0, -1e10)
            lp = torch.distributions.Categorical(logits=z).log_prob(t['actions'].long())
            ratio = torch.exp(lp - t['log_pi_old'])
            if it == 1:
                assert bool(((ratio < 0.95) | (ratio > 1.05)).all())
                v = model.values(t['obs'])
                orc.vn.update(t['returns'].reshape(-1, 1))
                d = (v - orc.vn.normalize(t['returns'].reshape(-1, 1)).reshape(-1)).abs()
                assert bool((d < 1.0).any()) and bool((d > 1.0).any())
                assert bool(((v - t['values']).abs() > 0.05).any())
                break
        orc.update(t['obs'], t['actions'], t['log_pi_old'], t['advantages'], t['values'], t['returns'],
                   t['agent_mask'].float(), t['avail_actions'])
    assert g["learner/infos"].shape == (3, 7)


def test_value_norm_float32_order_matches_torch():
    rng = np.random.default_rng(0)
    ref = ValueNormOracle()
    state = (np.float32(0), np.float32(0), np.float32(0))
    for _ in range(4):
        r = rng.normal(3.0, 5.0, 97).astype(np.float32)
        ref.update(torch.from_numpy(r).reshape(-1, 1))
        state, (mean, std) = value_norm_update_f32(*state, r, r.size)
        assert state[2] == ref.debiasing_term.item()
        m, var = ref.running_mean_var()
        # the batch moments are float64 quotients rounded once; torch sums in float32: a few ulp apart
        np.testing.assert_allclose(mean, m.item(), rtol=1e-5)
        np.testing.assert_allclose(std, np.sqrt(var.item()), rtol=1e-5)


def test_finish_path_reference_branches_agree_without_normaliser():
    rng = np.random.default_rng(1)
    rew, val = rng.normal(size=9).astype(np.float32), rng.normal(size=9).astype(np.float32)
    term = np.zeros(9, bool)
    term[-1] = True
    r1, a1 = finish_path_ref(rew, val, term, np.float32(0.0), True, 0.99, 1.0)
    r0, a0 = finish_path_ref(rew, val, term, np.float32(0.0), False, 0.99, 1.0)
    np.testing.assert_allclose(r1, r0, rtol=1e-5, atol=1e-5)    # lambda = 1: GAE returns are the discounted returns
    np.testing.assert_array_equal(a0, (r0 - val).astype(np.float32))


def test_mappo_entry_points_validate_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    j = ctypes.c_void_p(0x1000)
    EINVAL, ERANGE = -1, -3
    for name in ("xb_mappo_loss_fwd_bwd", "xb_mappo_prepare", "xb_value_norm_update", "xb_gae_scan_vn"):
        assert name in _lib.exported_symbols() and hasattr(lib, name)

    def k4m(R=8, A=7, R_total=8, avail=None, ld=0, old_value=j, vclip=0.2, mask=j, prep=j):
        return lib.xb_mappo_loss_fwd_bwd(j, avail, ld, j, j, j, j, old_value, j, mask, None, prep, R, A, R_total, 0.2,
                                         vclip, 10.0, 1.0, 0.01, j, j, j, j, None)
    assert k4m(A=65) == ERANGE
    assert k4m(R_total=4) == EINVAL
    assert k4m(A=0) == EINVAL and k4m(R=0) == EINVAL
    assert k4m(old_value=None) == EINVAL                      # value clipping needs the stored values
    assert k4m(avail=j, ld=6) == EINVAL                       # avail rows narrower than A
    assert k4m(mask=None) == EINVAL and k4m(prep=None) == EINVAL
    assert lib.xb_mappo_prepare(j, j, 0, j, j, None) == EINVAL
    assert lib.xb_mappo_prepare(None, j, 8, j, j, None) == EINVAL
    assert lib.xb_value_norm_update(j, j, j, j, 0, 0.99999, j, None) == EINVAL
    assert lib.xb_value_norm_update(j, j, j, j, 8, 1.0, j, None) == EINVAL
    assert lib.xb_value_norm_update(j, j, None, j, 8, 0.99999, j, None) == EINVAL
    assert lib.xb_gae_scan_vn(j, j, j, j, j, None, None, j, j, 0, 8, 0.99, 0.95, 1, None, None, None, None) == EINVAL
    assert lib.xb_gae_scan_vn(j, j, j, j, j, None, None, j, j, 4, 8, 0.99, 0.95, 1, j, None, None, None) == EINVAL


def _cfg(**over):
    from xuance_b200.common.common_tools import get_arguments
    d = dict(vars(get_arguments("mappo", "sc2", config_path=MAPPO_CONFIG)))
    d.update(dict(device="cpu"))
    d.update(over)
    return Namespace(**d)


def test_mappo_config_defines_every_key_the_classes_read():
    cfg = _cfg()
    for k in ("agent", "learner", "representation", "representation_hidden_size", "actor_hidden_size",
              "critic_hidden_size", "activation", "use_parameter_sharing", "use_actions_mask", "use_rnn", "seed",
              "parallels", "buffer_size", "n_epochs", "n_minibatch", "learning_rate", "vf_coef", "ent_coef",
              "clip_range", "gamma", "use_linear_lr_decay", "end_factor_lr_decay", "use_global_state",
              "use_value_clip", "value_clip_range", "use_value_norm", "use_huber_loss", "huber_delta", "use_advnorm",
              "use_gae", "gae_lambda", "use_grad_clip", "grad_clip_norm", "running_steps"):
        assert hasattr(cfg, k), k
    assert cfg.agent == "MAPPO" and cfg.learner == "MAPPO_Learner" and cfg.use_rnn is False
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    assert "MAPPO" in REGISTRY_Agents and "MAPPO_Learner" in REGISTRY_Learners


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import REGISTRY_Agents
    keys = ["agent_0", "agent_1"]
    obs = {k: Box(-1, 1, (12,), np.float32) for k in keys}
    disc = {k: Discrete(7) for k in keys}
    kw = dict(num_agents=2, agent_keys=keys, observation_space=obs, action_space=disc)
    with pytest.raises(NotImplementedError, match="use_rnn"):
        REGISTRY_Agents["MAPPO"](_cfg(use_rnn=True), **kw)
    with pytest.raises(NotImplementedError, match="use_parameter_sharing"):
        REGISTRY_Agents["MAPPO"](_cfg(use_parameter_sharing=False), **kw)
    with pytest.raises(NotImplementedError, match="Box"):
        REGISTRY_Agents["MAPPO"](_cfg(), num_agents=2, agent_keys=keys, observation_space=obs,
                                 action_space={k: Box(-1, 1, (2,), np.float32) for k in keys})
    with pytest.raises(NotImplementedError, match="IPPO"):
        REGISTRY_Agents["IPPO"](_cfg(agent="IPPO"), **kw)

"""CPU tests of the PPG stack: the float64 K4P restatements (tests/ppg_refs.py) against torch autograd of the reference's
expressions (q = 0 and p = 0 terms, -inf logits, new == old, A = 1, D = 1, the B*D mean of the Gaussian KL), the C-ABI
argument checks, no spills in the new kernels, the shipped configs and their lookup, the static config-key check, the
PhasicActorCritic parameter names, and the out-of-scope errors."""
import ctypes
import os
import re
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ppg_refs import (cat_aux_ref, gauss_aux_ref, torch_cat_aux_loss, torch_gauss_aux_loss, cat_batch,  # noqa: E402
                      gauss_batch)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _t(x, grad=False):
    return torch.tensor(np.asarray(x, np.float64), requires_grad=grad)


def _autograd_cat(z, o, v, aux, ret, kl_beta):
    zt, vt, at = _t(z, True), _t(v, True), _t(aux, True)
    loss, a_l, kl_l, v_l = torch_cat_aux_loss(zt, _t(o), vt, at, _t(ret), kl_beta)
    loss.backward()
    return zt.grad.numpy(), vt.grad.numpy(), at.grad.numpy(), [a_l.item(), kl_l.item(), v_l.item(), loss.item()]


@pytest.mark.parametrize("B,A", [(37, 5), (20, 1), (9, 64), (16, 2)])
def test_cat_reference_matches_autograd(B, A):
    rng = np.random.default_rng(B + A)
    z, o, v, aux, ret = cat_batch(rng, B, A)
    dz, dv, da, st, kl = cat_aux_ref(z, o, v, aux, ret, 0.8)
    gz, gv, ga, losses = _autograd_cat(z, o, v, aux, ret, 0.8)
    np.testing.assert_allclose(dz, gz, rtol=1e-10, atol=1e-16)
    np.testing.assert_allclose(dv, gv, rtol=1e-12)
    np.testing.assert_allclose(da, ga, rtol=1e-12)
    np.testing.assert_allclose(st[:4], losses, rtol=1e-12)
    want_kl = torch.distributions.kl_divergence(torch.distributions.Categorical(logits=_t(z)),
                                                torch.distributions.Categorical(logits=_t(o))).numpy()
    np.testing.assert_allclose(kl, want_kl, rtol=1e-12)
    if A > 1:
        assert np.isinf(kl[1]) and np.isinf(st[1])           # q = 0 under p > 0: +inf
        assert np.isfinite(kl[0]) and np.isfinite(dz).all()  # p = 0: the term is 0, and masked terms pass no gradient
    else:
        assert (kl == 0).all() and (dz == 0).all()           # one action: p = q = 1


def test_cat_reference_nan_rows_and_equal_distributions():
    rng = np.random.default_rng(1)
    z, o, v, aux, ret = cat_batch(rng, 6, 4, zeros=False)
    z[0, 1] = -np.inf
    o[1, 2] = -np.inf
    o[2] = z[2]
    dz, _, _, _, kl = cat_aux_ref(z, o, v, aux, ret, 1.0)
    gz, _, _, _ = _autograd_cat(z, o, v, aux, ret, 1.0)
    np.testing.assert_allclose(dz, gz, rtol=1e-10, atol=1e-16)         # equal_nan: the NaN rows are torch's
    assert np.isnan(dz[0]).all() and np.isnan(dz[1]).all() and np.isfinite(dz[2:]).all()
    assert kl[2] == 0.0 and np.abs(dz[2]).max() < 1e-17
    assert np.isinf(kl[1]) and np.isfinite(kl[0])


@pytest.mark.parametrize("B,D", [(37, 3), (20, 1), (9, 64), (5, 6)])
def test_gauss_reference_matches_autograd(B, D):
    rng = np.random.default_rng(B * D)
    mu, ls, omu, ols, v, aux, ret = gauss_batch(rng, B, D)
    dmu, dls, dv, da, st, kl = gauss_aux_ref(mu, ls, omu, ols, v, aux, ret, 0.6)
    mt, lt, vt, at = _t(mu, True), _t(ls, True), _t(v, True), _t(aux, True)
    loss, a_l, kl_l, v_l = torch_gauss_aux_loss(mt, lt, _t(omu), _t(ols).exp().expand(B, D), vt, at, _t(ret), 0.6)
    loss.backward()
    np.testing.assert_allclose(dmu, mt.grad.numpy(), rtol=1e-10, atol=1e-18)
    np.testing.assert_allclose(dls, lt.grad.numpy(), rtol=1e-10, atol=1e-16)
    np.testing.assert_allclose(dv, vt.grad.numpy(), rtol=1e-12)
    np.testing.assert_allclose(da, at.grad.numpy(), rtol=1e-12)
    np.testing.assert_allclose(st[:4], [a_l.item(), kl_l.item(), v_l.item(), loss.item()], rtol=1e-12)
    assert kl.shape == (B, D)                                 # a plain Normal: the KL is per component ...
    assert st[1] == pytest.approx(kl.sum() / (B * D), rel=1e-14)  # ... and the mean runs over B * D
    if D > 1:
        assert st[1] != pytest.approx(kl.sum() / B, rel=1e-3)
    same = gauss_aux_ref(mu, ls, mu, ls, v, aux, ret, 0.6)
    assert (same[5] == 0).all() and (same[0] == 0).all() and (same[1] == 0).all()


def test_ppg_entry_points_validate_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    j = ctypes.c_void_p(0x1000)
    EINVAL, ERANGE = -1, -3
    for name in ("xb_ppg_aux_loss_fwd_bwd", "xb_ppg_aux_gauss_loss_fwd_bwd"):
        assert name in _lib.exported_symbols() and hasattr(lib, name)

    def cat(B=8, A=4, Bt=8, z=j, o=j, v=j, aux=j, r=j, dz=j, dv=j, da=j, st=j, sc=j):
        return lib.xb_ppg_aux_loss_fwd_bwd(z, o, v, aux, r, B, A, Bt, 1.0, dz, dv, da, st, sc, None)

    def gauss(B=8, D=3, Bt=8, mu=j, ls=j, omu=j, ols=j, v=j, aux=j, r=j, dmu=j, dls=j, dv=j, da=j, st=j, sc=j):
        return lib.xb_ppg_aux_gauss_loss_fwd_bwd(mu, ls, omu, ols, v, aux, r, B, D, Bt, 1.0, dmu, dls, dv, da, st, sc,
                                                 None)
    for f in (cat, gauss):
        assert f(B=0) == EINVAL and f(B=-1, Bt=-1) == EINVAL and f(Bt=4) == EINVAL
    for k in ("v", "r", "dv", "st", "sc", "z", "o", "dz", "aux", "da"):
        assert cat(**{k: None}) == EINVAL, k
    assert cat(A=0) == EINVAL and cat(A=65) == ERANGE
    # every call above fails validation before any launch (the pointers are not device memory); that the critic-only
    # form ignores A is checked on the GPU with real buffers (test_gpu_ppg.py::test_cat_kernel_critic_only_form)
    assert cat(A=65, z=None, o=None, dz=None, Bt=4) == EINVAL
    for k in ("mu", "ls", "omu", "ols", "v", "aux", "r", "dmu", "dls", "dv", "da", "st", "sc"):
        assert gauss(**{k: None}) == EINVAL, k
    assert gauss(D=0) == EINVAL and gauss(D=65) == ERANGE
    # the Gaussian entry takes no workspace: its log_std gradient is one term per column times B (include/xb200.h), so
    # there is no workspace size to validate


def test_ppg_kernels_do_not_spill():
    from xuance_b200 import build
    log = open(os.path.join(os.path.dirname(build.__file__), "build.log")).read()
    entries = re.findall(r"Function properties for (\w+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", log)
    ppg = {e[0]: e[1:] for e in entries if "ppg_aux" in e[0]}
    assert len(ppg) == 4, sorted(ppg)
    for name, sizes in ppg.items():
        assert sizes == ("0", "0", "0"), (name, sizes)


def _cfg(env_id="CartPole-v1", **over):
    from xuance_b200.common.common_tools import get_arguments
    d = dict(vars(get_arguments("ppg", "classic_control", env_id)))
    d.update(device="cpu", **over)
    return Namespace(**d)


def test_configs_resolve_with_the_reference_values():
    import yaml
    from xuance_b200.common import common_tools
    root = os.path.join(ROOT, "xuance_b200", "configs", "ppg")
    assert not [f for f in os.listdir(root) if f.endswith(".yaml")]      # one directory below configs/ppg/ only
    for env_id, policy in (("CartPole-v1", "Categorical_PPG"), ("Pendulum-v1", "Gaussian_PPG")):
        path = os.path.join(root, "classic_control", env_id + ".yaml")
        cfg = vars(common_tools.get_arguments("ppg", "classic_control", env_id))
        for k, v in yaml.safe_load(open(path)).items():
            assert cfg[k] == v, (env_id, k)
        assert (cfg["agent"], cfg["learner"], cfg["policy"]) == ("PPG", "PPG_Learner", policy)
        assert (cfg["policy_nepoch"], cfg["value_nepoch"], cfg["aux_nepoch"], cfg["kl_beta"]) == (4, 8, 8, 1.0)
    for env, env_id in (("classic_control", "Acrobot-v1"), ("classic_control", "MountainCar-v0"),
                        ("box2d", "LunarLander-v3"), ("box2d", "BipedalWalker-v3"), ("mujoco", "Ant-v4")):
        with pytest.raises(AttributeError, match="no config"):
            common_tools.get_arguments("ppg", env, env_id)


def test_configs_define_every_key_their_classes_read():
    """Every ``config.X`` that ppg_agent.py, ppg_learner.py and their bases read without a getattr / hasattr default is a
    key of basic.yaml + the yaml."""
    import yaml
    root = os.path.join(ROOT, "xuance_b200")
    rd = lambda *p: open(os.path.join(root, *p)).read()
    base = set(yaml.safe_load(rd("configs", "basic.yaml")))
    src = "".join(rd(*f.split("/")) for f in ["torch/agents/ppg_agent.py", "torch/agents/ppo_agent.py",
                                             "torch/agents/on_policy.py", "torch/agents/agent.py",
                                             "torch/learners/ppg_learner.py", "torch/learners/learner.py"])
    hard = set(re.findall(r"(?<![a-zA-Z_])(?:self\.)?config\.([a-zA-Z_][a-zA-Z0-9_]*)\b(?!\s*=[^=])", src))
    soft = set(re.findall(r"(?:getattr|hasattr)\((?:self\.)?config,\s*.([a-zA-Z_0-9]+).", src))
    for env_id in ("CartPole-v1", "Pendulum-v1"):
        cfg = yaml.safe_load(open(os.path.join(root, "configs", "ppg", "classic_control", env_id + ".yaml")))
        assert not sorted(hard - soft - base - set(cfg)), env_id
    assert {"policy_nepoch", "value_nepoch", "aux_nepoch", "kl_beta"} <= hard


def test_phasic_actor_critic_parameter_names():
    """The reference's PhasicActorCritic names (actor.representation / actor.actor_head, critic.representation /
    critic.critic_head, aux_critic.*), the three groups in that order, and three independent deep copies of one
    representation."""
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents.ppg_agent import PPG_Agent
    obs = Box(-1, 1, (4,), np.float32)
    for act in (Discrete(3), Box(-1, 1, (2,), np.float32)):
        env_id = "CartPole-v1" if isinstance(act, Discrete) else "Pendulum-v1"
        agent = PPG_Agent.__new__(PPG_Agent)
        from xuance_b200.torch.agents.agent import Agent
        Agent.__init__(agent, _cfg(env_id), None, obs, act)
        model = agent._build_model()
        keys = list(model.state_dict())
        head = "actor.actor_head.logits." if isinstance(act, Discrete) else "actor.actor_head.mu."
        assert keys[0].startswith("actor.representation.") and any(k.startswith(head) for k in keys)
        if not isinstance(act, Discrete):
            assert "actor.actor_head.log_std" in keys
        assert any(k.startswith("critic.critic_head.values.") for k in keys)
        assert any(k.startswith("aux_critic.critic_head.values.") for k in keys)
        order = [k.split(".")[0] for k in keys]
        assert order == sorted(order, key=["actor", "critic", "aux_critic"].index)
        sd = model.state_dict()
        for k in [k for k in keys if k.startswith("actor.representation.")]:
            assert torch.equal(sd[k], sd["critic" + k[5:]]) and torch.equal(sd[k], sd["aux_critic" + k[5:]])
            assert sd[k].data_ptr() != sd["critic" + k[5:]].data_ptr()
        model.load_state_dict({k: v.clone() for k, v in sd.items()}, strict=True)


def test_registries():
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    assert REGISTRY_Agents["PPG"].__name__ == "PPG_Agent" and "PPG_Learner" in REGISTRY_Learners


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import REGISTRY_Agents
    obs = Box(-1, 1, (4,), np.float32)
    with pytest.raises(NotImplementedError, match="action masks"):
        REGISTRY_Agents["PPG"](_cfg(use_actions_mask=True), observation_space=obs, action_space=Discrete(2))
    with pytest.raises(NotImplementedError, match="at most 64 actions"):
        REGISTRY_Agents["PPG"](_cfg(), observation_space=obs, action_space=Discrete(65))
    with pytest.raises(NotImplementedError, match="at most 64 action components"):
        REGISTRY_Agents["PPG"](_cfg("Pendulum-v1"), observation_space=obs, action_space=Box(-1, 1, (65,), np.float32))
    with pytest.raises(NotImplementedError, match="Discrete and one-dimensional Box"):
        REGISTRY_Agents["PPG"](_cfg("Pendulum-v1"), observation_space=obs, action_space=Box(-1, 1, (2, 3), np.float32))


# ====================================================================================================== reference fixture
GOLDEN = os.path.join(HERE, "golden", "ppg_update.npz")


def _fixture_model(g, pre, kind, device="cpu"):
    from oracle_ppg import build_fixture_model
    model = build_fixture_model(kind, device)
    init = {k[len(pre + "init/"):]: torch.from_numpy(g[k]) for k in g.files if k.startswith(pre + "init/")}
    # strict load of the reference's state_dict, and ours is exactly the reference's (names, order, shapes, dtypes):
    # each loads into the other with strict=True
    model.load_state_dict(init, strict=True)
    ours = model.state_dict()
    assert list(ours) == list(init)
    for k in ours:
        assert ours[k].shape == init[k].shape and ours[k].dtype == init[k].dtype, k
    return model


@pytest.mark.parametrize("kind,mb,clip", [(k, m, c) for k in ("cat", "gauss") for m in (1, 2) for c in (0, 1)])
def test_oracle_matches_reference_fixture(kind, mb, clip):
    """The torch oracle on this package's model classes replays the reference's full cycle (three phases and the
    relabel) and lands on the reference's infos, parameters and per-parameter Adam state after every phase."""
    from oracle_ppg import PPGOracle
    from ppg_refs import FIX_INFO_KEYS, fix_learner_config
    g = np.load(GOLDEN)
    pre = f"{kind}/mb{mb}/clip{clip}/"
    model = _fixture_model(g, pre, kind)
    c = fix_learner_config(mb, clip)
    orc = PPGOracle(model, c["learning_rate"], c["ent_coef"], c["clip_range"], c["kl_beta"], c["use_grad_clip"],
                    c["grad_clip_norm"], c["end_factor_lr_decay"], int(g[pre + "total_iters"]))
    t = lambda k: torch.from_numpy(g[pre + "in/" + k])
    obs, act, adv, ret, old_logp = t("obs"), t("actions"), t("advantages"), t("returns"), t("old_logp")
    act = act if kind == "gauss" else act.long()
    names = {id(p): n for n, p in model.named_parameters()}
    for phase in ("actor", "critic", "aux"):
        if phase == "aux":
            old = orc.relabel(obs)
            if kind == "gauss":
                np.testing.assert_allclose(old[0].numpy(), g[pre + "relabel/mu"], rtol=1e-6, atol=1e-7)
                np.testing.assert_allclose(old[1].numpy(), g[pre + "relabel/std"], rtol=1e-6)   # one [D] scale
            else:
                np.testing.assert_allclose(old[0].numpy(), g[pre + "relabel/logits"], rtol=1e-6, atol=1e-7)
        for n, idx in enumerate(g[f"{pre}idx/{phase}"]):
            idx = torch.from_numpy(idx)
            if phase == "actor":
                info = orc.update_actor(obs[idx], act[idx], adv[idx], old_logp[idx])
            elif phase == "critic":
                info = orc.update_critic(obs[idx], ret[idx])
            else:
                info = orc.update_auxiliary_critic(obs[idx], ret[idx], (old[0][idx], old[1]) if kind == "gauss"
                                                   else (old[0][idx],))
            np.testing.assert_allclose([info[k] for k in FIX_INFO_KEYS[phase]], g[f"{pre}info/{phase}"][n], rtol=1e-5,
                                       atol=1e-7, err_msg=f"{phase} {n}")
        after = f"{pre}after/{phase}/"
        for k, v in model.state_dict().items():
            np.testing.assert_allclose(v.numpy(), g[after + k], rtol=1e-5, atol=1e-6, err_msg=f"{phase} {k}")
        stepped = {n for n, p in model.named_parameters() if p in orc.optimizer.state}
        assert stepped == {k[len(after + "adam/"):].split("/")[0] for k in g.files if k.startswith(after + "adam/")}, phase
        for p, st in orc.optimizer.state.items():
            n = names[id(p)]
            assert float(st["step"]) == float(g[f"{after}adam/{n}/step"]), (phase, n)
            for m in ("exp_avg", "exp_avg_sq"):
                np.testing.assert_allclose(st[m].numpy(), g[f"{after}adam/{n}/{m}"], rtol=1e-4, atol=1e-9,
                                           err_msg=f"{phase} {n} {m}")


def test_reference_fixture_covers_the_quirks():
    """Each group's Adam step follows the phases its loss reaches, the LinearLR schedule moves only in the policy
    phase, and the clip binds in the clipped cases."""
    from ppg_refs import FIX_LR
    g = np.load(GOLDEN)
    for kind in ("cat", "gauss"):
        for mb in (1, 2):
            pre = f"{kind}/mb{mb}/clip0/"
            step = lambda ph, n: float(g[f"{pre}after/{ph}/adam/{n}/step"])
            assert not [k for k in g.files if k.startswith(pre + "after/actor/adam/critic")]
            assert step("actor", "actor.representation.model.0.weight") == 2 * mb
            assert step("critic", "critic.representation.model.0.weight") == 2 * mb
            assert not [k for k in g.files if k.startswith(pre + "after/critic/adam/aux_critic")]
            assert step("aux", "actor.representation.model.0.weight") == 4 * mb
            assert step("aux", "aux_critic.representation.model.0.weight") == 2 * mb
            lr = g[pre + "info/actor"][:, 2]              # logged after each scheduler step: down to end_factor 0.5
            assert (np.diff(lr) < 0).all() and lr[-1] == pytest.approx(0.5 * FIX_LR)
            d = lambda c: np.abs(g[f"{kind}/mb{mb}/clip{c}/after/actor/actor.representation.model.0.weight"]
                                 - g[f"{kind}/mb{mb}/clip{c}/init/actor.representation.model.0.weight"]).max()
            assert d(1) < d(0)

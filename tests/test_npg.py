"""CPU tests of the NPG stack: the float64 K4N restatements (tests/npg_refs.py) against torch autograd of the reference's
expressions (A = 1, D = 1, p = 0 for an untaken action, positive Gaussian log-densities), K7N's closed form against a
float64 dense inverse of the reference's F (kappa = 0, > 0, < 0, next to the pole), the torch oracle against every
update of the reference fixture, the C-ABI argument checks, no spills in the new kernels, the shipped configs, the
registries and the out-of-scope errors."""
import ctypes
import os
import re
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from npg_refs import (cat_ref, gauss_ref, torch_npg_terms, natural_grad_ref, dense_ref, conditioning,  # noqa: E402
                      FIX_CASES, FIX_INFO_KEYS, fix_learner_config)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EPS32 = 2.0 ** -23


def _t(x, grad=False):
    return torch.tensor(np.asarray(x, np.float64), requires_grad=grad)


def _autograd(out, v, act, adv, ret, gaussian):
    """(d a_loss / d outputs, d sum log pi / d outputs, d c_loss / d v, [a_loss, c_loss, sum log pi]) by autograd."""
    vt = _t(v, True)
    lp_sum, a_loss, c_loss = torch_npg_terms(out, vt, _t(act), _t(adv), _t(ret), gaussian)
    ins = list(out) if gaussian else [out]
    loss_g = torch.autograd.grad(a_loss, ins, retain_graph=True)
    score_g = torch.autograd.grad(lp_sum, ins)
    (dv,) = torch.autograd.grad(c_loss, vt)
    return ([x.numpy() for x in loss_g], [x.numpy() for x in score_g], dv.numpy(),
            [a_loss.item(), c_loss.item(), lp_sum.item()])


@pytest.mark.parametrize("B,A", [(37, 5), (20, 1), (9, 64), (16, 2)])
def test_cat_reference_matches_autograd(B, A):
    rng = np.random.default_rng(B + A)
    z = rng.normal(size=(B, A)) * 2
    act = rng.integers(0, A, B).astype(np.float32)
    if A > 1:                                       # p = 0 for an untaken action (underflows in float64 too)
        z[0, (int(act[0]) + 1) % A] -= 1e4
    v, adv, ret = rng.normal(size=B), rng.normal(size=B), rng.normal(size=B)
    dz, sz, dv, st, lps = cat_ref(z, v, act, adv, ret)
    (gz,), (gs,), gv, losses = _autograd(_t(z, True), v, act, adv, ret, False)
    np.testing.assert_allclose(dz, gz, rtol=1e-12, atol=1e-18)
    np.testing.assert_allclose(sz, gs, rtol=1e-12, atol=1e-18)
    np.testing.assert_allclose(dv, gv, rtol=1e-12)
    np.testing.assert_allclose([st[0], st[1], lps], losses, rtol=1e-12)
    assert st[3] == lps and st[2] == pytest.approx(v.mean(), rel=1e-14)
    if A == 1:
        assert (sz == 0).all() and lps == 0.0       # one action: log pi = 0, no score
    else:
        assert sz[0, (int(act[0]) + 1) % A] == 0.0


@pytest.mark.parametrize("B,D", [(37, 3), (20, 1), (9, 64), (5, 6)])
def test_gauss_reference_matches_autograd(B, D):
    rng = np.random.default_rng(B * D)
    mu = rng.normal(size=(B, D))
    ls = rng.normal(size=D) * 0.3 - 0.5
    x = mu + rng.normal(size=(B, D)) * np.exp(ls)
    v, adv, ret = rng.normal(size=B), rng.normal(size=B), rng.normal(size=B)
    dmu, dls, smu, sls, dv, st, lps = gauss_ref(mu, ls, v, x, adv, ret)
    (gmu, gls), (hmu, hls), gv, losses = _autograd((_t(mu, True), _t(ls, True)), v, x, adv, ret, True)
    np.testing.assert_allclose(dmu, gmu, rtol=1e-12, atol=1e-18)
    np.testing.assert_allclose(dls, gls, rtol=1e-10, atol=1e-15)
    np.testing.assert_allclose(smu, hmu, rtol=1e-12, atol=1e-18)
    np.testing.assert_allclose(sls, hls, rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(dv, gv, rtol=1e-12)
    np.testing.assert_allclose([st[0], st[1], lps], losses, rtol=1e-11)


def test_gauss_reference_positive_log_densities():
    """Narrow Gaussians at their means have log pi > 0, so kappa = sum log pi / horizon_size > 0 (F is then positive
    definite, where the usual case kappa < 0 makes it indefinite)."""
    rng = np.random.default_rng(3)
    B, D = 12, 2
    mu = rng.normal(size=(B, D))
    ls = np.full(D, -3.0)
    x = mu + rng.normal(size=(B, D)) * 0.1 * np.exp(ls)
    v, adv, ret = rng.normal(size=B), rng.normal(size=B), rng.normal(size=B)
    *_, lps = gauss_ref(mu, ls, v, x, adv, ret)
    _, _, _, losses = _autograd((_t(mu, True), _t(ls, True)), v, x, adv, ret, True)
    assert lps > 0 and losses[2] == pytest.approx(lps, rel=1e-12)


@pytest.mark.parametrize("P", [1, 7, 300])
@pytest.mark.parametrize("regime", ["zero", "positive", "negative", "pole"])
def test_closed_form_matches_dense_inverse(P, regime):
    """Sherman-Morrison against torch.linalg.inv of the reference's F = kappa s s^T + lam I in float64.  Next to the pole
    (lam + kappa s.s within 1 % of 0) F is nearly singular; the dense inverse loses digits in proportion to the
    conditioning ratio, and the tolerance scales with it."""
    rng = np.random.default_rng(P)
    g, s = rng.normal(size=P), rng.normal(size=P)
    ss = s @ s
    kappa = {"zero": 0.0, "positive": 0.7, "negative": -0.9, "pole": -1e-3 / ss * 1.006}[regime]
    r = conditioning(s, kappa)
    got, want = natural_grad_ref(g, s, kappa), dense_ref(g, s, kappa)
    tol = 64 * 2.0 ** -52 * max(1.0, abs(r)) * P
    assert np.abs(got - want).max() <= tol * np.abs(want).max(), (regime, r)
    if regime == "zero":
        np.testing.assert_allclose(got, g / 1e-3, rtol=1e-15)
    if regime == "pole":
        assert 0 < abs(r) < 0.01 * abs(kappa * ss / 1e-3) and abs(r) < 0.01


def test_closed_form_is_the_inverse():
    """F (F^-1 g) = g for the closed form, in float64, including a kappa whose F is indefinite."""
    rng = np.random.default_rng(9)
    g, s = rng.normal(size=50), rng.normal(size=50)
    for kappa in (-3.0, 0.25):
        F = kappa * np.outer(s, s) + 1e-3 * np.eye(50)
        np.testing.assert_allclose(F @ natural_grad_ref(g, s, kappa), g, rtol=1e-9, atol=1e-12)


# ====================================================================================================== reference fixture
GOLDEN = os.path.join(HERE, "golden", "npg_update.npz")


def _fixture_model(g, pre, kind, device="cpu"):
    from oracle_npg import build_fixture_model
    model = build_fixture_model(kind, device)
    init = {k[len(pre + "init/"):]: torch.from_numpy(g[k]) for k in g.files if k.startswith(pre + "init/")}
    # strict load of the reference's state_dict, and ours is exactly the reference's (names, order, shapes, dtypes)
    model.load_state_dict(init, strict=True)
    ours = model.state_dict()
    assert list(ours) == list(init)
    for k in ours:
        assert ours[k].shape == init[k].shape and ours[k].dtype == init[k].dtype, k
    return model


def load_fixture_state(g, pre, model, opts):
    """The reference's parameters and both optimisers' Adam state after an update, into ``model`` and torch Adams."""
    with torch.no_grad():
        for k, v in model.state_dict().items():
            v.copy_(torch.from_numpy(g[pre + k]))
    names = {id(p): n for n, p in model.named_parameters()}
    for o in opts:
        for p in o.param_groups[0]["params"]:
            n = names[id(p)]
            o.state[p] = {"step": torch.tensor(float(g[f"{pre}adam/{n}/step"])),
                          "exp_avg": torch.from_numpy(g[f"{pre}adam/{n}/exp_avg"]).to(p.device).clone(),
                          "exp_avg_sq": torch.from_numpy(g[f"{pre}adam/{n}/exp_avg_sq"]).to(p.device).clone()}


def natgrad_tolerance(ratio):
    """The reference inverts F in float32: its F^-1 g is off by up to about |ratio| * eps32 of the vector's scale, where
    ratio = (lam + kappa s.s) / lam (the recorded conditioning; measured worst: 0.44 |ratio| eps32).  Four times the
    unit, with a floor at 1e-5 for well-conditioned tensors."""
    return max(1e-5, 4.0 * abs(ratio) * EPS32)


PARAM_ATOL = {"cat": 1e-4, "gauss": 5e-3}
# One Adam step moves each parameter by up to about lr = 1e-2 whatever its gradient's size, so a component of the
# reference's natural gradient that is within its float32 error of zero can move either way.  The Categorical fixture's
# ratios stay below 2.5e4 (error <= 1.5e-3 of scale), the Gaussian's reach 2.8e6 (error <= 0.17 of scale): measured
# worst parameter differences per update 1e-4 and 3.8e-3.


@pytest.mark.parametrize("kind,mb,clip", FIX_CASES)
def test_oracle_matches_reference_fixture(kind, mb, clip):
    """The torch oracle on this package's model classes, started from the reference's state before each update, lands on
    its infos, its post-clip natural gradient per actor tensor (tolerance from the recorded conditioning ratio), its
    Adam moments and its parameters."""
    from oracle_npg import NPGOracle
    g = np.load(GOLDEN)
    pre = f"{kind}/mb{mb}/clip{clip}/"
    model = _fixture_model(g, pre, kind)
    c = fix_learner_config(mb, clip)
    orc = NPGOracle(model, c["learning_rate"], c["use_grad_clip"], c["grad_clip_norm"], c["end_factor_lr_decay"],
                    c["running_steps"], c["horizon_size"])
    t = lambda k: torch.from_numpy(g[pre + "in/" + k])
    obs, act, adv, ret = t("obs"), t("actions"), t("advantages"), t("returns")
    act = act if kind == "gauss" else act.long()
    names = list(g[pre + "actor_names"])
    assert names == [n for n, _ in model.actor.named_parameters(prefix="actor")]
    for u, idx in enumerate(g[pre + "idx"]):
        if u:
            load_fixture_state(g, f"{pre}after{u - 1}/", model, [orc.actor_optimizer, orc.critic_optimizer])
        i = torch.from_numpy(idx)
        info = orc.update(obs[i], act[i], ret[i], adv[i])
        np.testing.assert_allclose([info[k] for k in FIX_INFO_KEYS], g[pre + "info"][u], rtol=1e-5, atol=1e-7)
        after = f"{pre}after{u}/"
        assert orc.kappa == pytest.approx(g[pre + "fisher"][u, 0, 0], rel=1e-6)
        for j, n in enumerate(names):
            want = g[f"{after}natgrad/{n}"]
            tol = natgrad_tolerance(g[pre + "fisher"][u, j, 1]) * np.abs(want).max()
            assert np.abs(orc.natural_grads[j].numpy() - want).max() <= tol, (u, n)
            for m, w in (("exp_avg", 0.1), ("exp_avg_sq", None)):
                ref = g[f"{after}adam/{n}/{m}"]
                p = dict(model.named_parameters())[n]
                got = orc.actor_optimizer.state[p][m].numpy()
                if w is not None:       # (1 - beta1) of this update's natural gradient error, on top of float32 rounding
                    assert np.abs(got - ref).max() <= w * tol + 1e-6 * np.abs(ref).max(), (u, n, m)
        for k, v in model.state_dict().items():
            np.testing.assert_allclose(v.numpy(), g[after + k], rtol=0, atol=PARAM_ATOL[kind], err_msg=f"{u} {k}")
            if k.startswith("critic."):             # the critic's step has no natural gradient: tight
                np.testing.assert_allclose(v.numpy(), g[after + k], rtol=1e-5, atol=1e-6, err_msg=f"{u} {k}")


def test_reference_fixture_records_the_quirks():
    """The unmodified learner raised AttributeError on ``.distribution``; kappa divides by horizon_size, not B; the
    critic's logged learning rate is the actor's; the Gaussian fixture's F is indefinite and badly conditioned."""
    g = np.load(GOLDEN)
    assert "AttributeError" in str(g["unpatched_error"]) and "'distribution'" in str(g["unpatched_error"])
    for kind, mb, clip in FIX_CASES:
        pre = f"{kind}/mb{mb}/clip{clip}/"
        info = g[pre + "info"]
        assert (info[:, 2] == info[:, 3]).all()
        assert info[-1, 2] == pytest.approx(0.5 * fix_learner_config(mb, clip)["learning_rate"])
        assert (g[pre + "fisher"][:, :, 0] < 0).all()     # sum log pi < 0 -> kappa < 0 -> F indefinite
    assert np.abs(g["gauss/mb1/clip0/fisher"][:, :, 1]).max() > 1e5


# ====================================================================================================== ABI
def test_npg_entry_points_validate_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    j = ctypes.c_void_p(0x1000)
    EINVAL, ERANGE = -1, -3
    for name in ("xb_npg_loss_fwd_bwd", "xb_npg_gauss_loss_fwd_bwd", "xb_npg_gauss_ws_doubles", "xb_npg_segment_table",
                 "xb_npg_natural_grad"):
        assert name in _lib.exported_symbols() and hasattr(lib, name)

    def cat(B=8, A=4, z=j, v=j, a=j, ad=j, r=j, dz=j, sz=j, dv=j, st=j, ls=j, sc=j):
        return lib.xb_npg_loss_fwd_bwd(z, v, a, ad, r, B, A, dz, sz, dv, st, ls, sc, None)
    assert cat(B=0) == EINVAL and cat(A=0) == EINVAL and cat(A=65) == ERANGE
    for k in ("z", "v", "a", "ad", "r", "dz", "sz", "dv", "st", "ls", "sc"):
        assert cat(**{k: None}) == EINVAL, k

    need = lib.xb_npg_gauss_ws_doubles(1000, 3)
    assert need == 2 * 3 * 125 and lib.xb_npg_gauss_ws_doubles(1 << 40, 64) == 2 * 64 * 2048
    assert lib.xb_npg_gauss_ws_doubles(0, 3) == 0

    def gauss(B=1000, D=3, ws_n=need, **ptrs):
        p = {k: j for k in ("mu", "ls", "v", "x", "ad", "r", "dmu", "dls", "smu", "sls", "dv", "st", "lps", "sc", "ws")}
        p.update(ptrs)
        return lib.xb_npg_gauss_loss_fwd_bwd(p["mu"], p["ls"], p["v"], p["x"], p["ad"], p["r"], B, D, p["dmu"],
                                             p["dls"], p["smu"], p["sls"], p["dv"], p["st"], p["lps"], p["sc"],
                                             p["ws"], ws_n, None)
    assert gauss(B=0) == EINVAL and gauss(D=0) == EINVAL and gauss(D=65, ws_n=1 << 20) == ERANGE
    assert gauss(ws_n=need - 1) == EINVAL
    for k in ("mu", "ls", "v", "x", "ad", "r", "dmu", "dls", "smu", "sls", "dv", "st", "lps", "sc", "ws"):
        assert gauss(**{k: None}) == EINVAL, k

    def nat(nseg=2, nchunks=3, horizon=16.0, lam=1e-3, ws_n=6, g=j, s=j, t=j, lps=j, ws=j):
        return lib.xb_npg_natural_grad(g, s, t, nseg, nchunks, lps, horizon, lam, ws, ws_n, None)
    for k in ("g", "s", "t", "lps", "ws"):
        assert nat(**{k: None}) == EINVAL, k
    assert nat(nseg=0) == EINVAL and nat(nchunks=1) == EINVAL and nat(ws_n=5) == EINVAL
    assert nat(horizon=0.0) == EINVAL and nat(lam=0.0) == EINVAL and nat(lam=-1e-3) == EINVAL
    assert nat(nchunks=1 << 31, ws_n=1 << 33) == ERANGE


def test_segment_table():
    """{offset, length, first chunk} per segment, chunks of 4096 elements; zero-length segments are refused."""
    from xuance_b200 import _lib
    lib = _lib.load()
    off = np.array([0, 32, 8224, 8256], np.int64)
    lens = np.array([1, 8192, 4097, 3], np.int64)
    table = np.zeros(12, np.int64)
    n = lib.xb_npg_segment_table(off.ctypes.data, lens.ctypes.data, 4, table.ctypes.data)
    assert n == 1 + 2 + 2 + 1
    assert table.reshape(4, 3).tolist() == [[0, 1, 0], [32, 8192, 1], [8224, 4097, 3], [8256, 3, 5]]
    lens[2] = 0
    assert lib.xb_npg_segment_table(off.ctypes.data, lens.ctypes.data, 4, table.ctypes.data) == -1
    assert lib.xb_npg_segment_table(off.ctypes.data, lens.ctypes.data, 0, table.ctypes.data) == -1


def test_npg_kernels_do_not_spill():
    from xuance_b200 import build
    log = open(os.path.join(os.path.dirname(build.__file__), "build.log")).read()
    entries = re.findall(r"Function properties for (\w+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", log)
    npg = {e[0]: e[1:] for e in entries if re.search(r"npg_\w+_kernel", e[0])}
    assert len(npg) == 4, sorted(npg)
    for name, sizes in npg.items():
        assert sizes == ("0", "0", "0"), (name, sizes)


# ====================================================================================================== configs, scope
def _cfg(env_id="CartPole-v1", **over):
    from xuance_b200.common.common_tools import get_arguments
    d = dict(vars(get_arguments("npg", "classic_control", env_id)))
    d.update(device="cpu", **over)
    return Namespace(**d)


def test_configs_resolve_with_the_reference_values():
    import yaml
    from xuance_b200.common import common_tools
    root = os.path.join(ROOT, "xuance_b200", "configs", "npg")
    assert not [f for f in os.listdir(root) if f.endswith(".yaml")]      # one directory below configs/npg/ only
    for env_id, policy, hidden in (("CartPole-v1", "Categorical_AC", 128), ("Pendulum-v1", "Gaussian_AC", 256)):
        path = os.path.join(root, "classic_control", env_id + ".yaml")
        cfg = vars(common_tools.get_arguments("npg", "classic_control", env_id))
        for k, v in yaml.safe_load(open(path)).items():
            assert cfg[k] == v, (env_id, k)
        assert (cfg["agent"], cfg["learner"], cfg["policy"]) == ("NPG", "NPG_Learner", policy)
        assert cfg["representation_hidden_size"] == [hidden] and cfg["actor_hidden_size"] == [hidden]
    for env, env_id in (("classic_control", "Acrobot-v1"), ("classic_control", "MountainCar-v0"),
                        ("box2d", "LunarLander-v3"), ("box2d", "BipedalWalker-v3"), ("mujoco", "Ant-v4")):
        with pytest.raises(AttributeError, match="no config"):
            common_tools.get_arguments("npg", env, env_id)


def test_configs_define_every_key_their_classes_read():
    """Every ``config.X`` that npg_agent.py, npg_learner.py and their bases read without a getattr / hasattr default is a
    key of basic.yaml + the yaml."""
    import yaml
    root = os.path.join(ROOT, "xuance_b200")
    rd = lambda *p: open(os.path.join(root, *p)).read()
    base = set(yaml.safe_load(rd("configs", "basic.yaml")))
    src = "".join(rd(*f.split("/")) for f in ["torch/agents/npg_agent.py", "torch/agents/ppo_agent.py",
                                             "torch/agents/on_policy.py", "torch/agents/agent.py",
                                             "torch/learners/npg_learner.py", "torch/learners/learner.py"])
    hard = set(re.findall(r"(?<![a-zA-Z_])(?:self\.)?config\.([a-zA-Z_][a-zA-Z0-9_]*)\b(?!\s*=[^=])", src))
    soft = set(re.findall(r"(?:getattr|hasattr)\((?:self\.)?config,\s*.([a-zA-Z_0-9]+).", src))
    for env_id in ("CartPole-v1", "Pendulum-v1"):
        cfg = yaml.safe_load(open(os.path.join(root, "configs", "npg", "classic_control", env_id + ".yaml")))
        assert not sorted(hard - soft - base - set(cfg)), env_id
    assert {"horizon_size", "running_steps", "learning_rate", "critic_hidden_size"} <= hard


def _model(env_id, act_space):
    from xuance_b200.common import Box
    from xuance_b200.torch.agents.npg_agent import NPG_Agent
    from xuance_b200.torch.agents.agent import Agent
    agent = NPG_Agent.__new__(NPG_Agent)
    Agent.__init__(agent, _cfg(env_id), None, Box(-1, 1, (4,), np.float32), act_space)
    return agent, agent._build_model()


def test_model_is_the_reference_actor_critic():
    """ActorCritic(actor, critic) with the reference's names, the representation deep-copied into the critic, and the
    raw-output methods on ActorCritic."""
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.rl_models import ActorCritic, PhasicActorCritic
    for env_id, act in (("CartPole-v1", Discrete(3)), ("Pendulum-v1", Box(-1, 1, (2,), np.float32))):
        _, model = _model(env_id, act)
        assert type(model) is ActorCritic
        keys = list(model.state_dict())
        assert {k.split(".")[0] for k in keys} == {"actor", "critic"}
        head = "actor.actor_head.logits." if env_id == "CartPole-v1" else "actor.actor_head.mu."
        assert any(k.startswith(head) for k in keys)
        sd = model.state_dict()
        for k in [k for k in keys if k.startswith("actor.representation.")]:
            assert torch.equal(sd[k], sd["critic" + k[5:]]) and sd[k].data_ptr() != sd["critic" + k[5:]].data_ptr()
        obs = torch.zeros(5, 4)
        if env_id == "CartPole-v1":
            logits, v = model.forward_raw(obs)
            assert logits.shape == (5, 3) and v.shape == (5,)
        else:
            mu, log_std, v = model.forward_raw_gauss(obs)
            assert mu.shape == (5, 2) and log_std is model.actor.actor_head.log_std and v.shape == (5,)
    for name in ("logits", "mu_log_std", "forward_raw", "forward_raw_gauss"):
        assert name in vars(ActorCritic) and name not in vars(PhasicActorCritic)


def test_registries():
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    assert REGISTRY_Agents["NPG"].__name__ == "NPG_Agent" and REGISTRY_Learners["NPG_Learner"].__name__ == "NPG_Learner"


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import REGISTRY_Agents
    obs = Box(-1, 1, (4,), np.float32)
    with pytest.raises(NotImplementedError, match="action masks"):
        REGISTRY_Agents["NPG"](_cfg(use_actions_mask=True), observation_space=obs, action_space=Discrete(2))
    with pytest.raises(NotImplementedError, match="at most 64 actions"):
        REGISTRY_Agents["NPG"](_cfg(), observation_space=obs, action_space=Discrete(65))
    with pytest.raises(NotImplementedError, match="at most 64 action components"):
        REGISTRY_Agents["NPG"](_cfg("Pendulum-v1"), observation_space=obs, action_space=Box(-1, 1, (65,), np.float32))
    with pytest.raises(NotImplementedError, match="Discrete and one-dimensional Box"):
        REGISTRY_Agents["NPG"](_cfg("Pendulum-v1"), observation_space=obs, action_space=Box(-1, 1, (2, 3), np.float32))
    agent, _ = _model("CartPole-v1", Discrete(2))
    agent.world_size = 2                     # kappa, s and g would all need an all-reduce before K7N
    with pytest.raises(NotImplementedError, match="one GPU"):
        agent._build_model()

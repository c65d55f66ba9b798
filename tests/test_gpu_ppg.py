"""GPU: the K4P kernels against their float64 restatements (tests/ppg_refs.py) across row counts, action counts and the
zero-probability / NaN regimes, shard sums and launch-to-launch bit identity; PPG_Learner against the reference's own
update cycles (tests/golden/ppg_update.npz) and against the torch oracle (tests/oracle_ppg.py, on a deep copy of the
model) phase by phase, eager and as CUDA graphs; the per-group Adam leaving untouched groups alone; the buffer's
old-distribution field; and learning through REGISTRY_Agents["PPG"]."""
import copy
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ppg_refs import cat_aux_ref, gauss_aux_ref, cat_batch, gauss_batch  # noqa: E402
from oracle_ppg import PPGOracle  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BIG = 2048 * 256 + 5


def _d(x):
    return torch.as_tensor(np.ascontiguousarray(x), device=DEV)


def _cat_launch(z, o, v, aux, ret, kl_beta, B_total=None):
    from xuance_b200 import _lib
    B = len(v)
    A = 0 if z is None else z.shape[1]
    zd, od = (None, None) if z is None else (_d(z), _d(o))
    vd, rd = _d(v), _d(ret)
    ad = None if aux is None else _d(aux)
    dz = None if z is None else torch.empty_like(zd)
    dv = torch.empty_like(vd)
    da = None if aux is None else torch.empty_like(ad)
    st = torch.empty(8, dtype=torch.float32, device=DEV)
    sc = _lib.scratch(DEV)
    _lib.call("xb_ppg_aux_loss_fwd_bwd", _lib.ptr(zd), _lib.ptr(od), _lib.ptr(vd), _lib.ptr(ad), _lib.ptr(rd), B, A,
              B if B_total is None else B_total, float(kl_beta), _lib.ptr(dz), _lib.ptr(dv), _lib.ptr(da),
              _lib.ptr(st), _lib.ptr(sc))
    cpu = lambda t: None if t is None else t.cpu().numpy()
    return cpu(dz), cpu(dv), cpu(da), cpu(st)


def _gauss_launch(mu, ls, omu, ols, v, aux, ret, kl_beta, B_total=None):
    from xuance_b200 import _lib
    B, D = mu.shape
    ins = [_d(x) for x in (mu, ls, omu, ols, v, aux, ret)]
    dmu, dls = torch.empty_like(ins[0]), torch.empty_like(ins[1])
    dv, da = torch.empty_like(ins[4]), torch.empty_like(ins[5])
    st = torch.empty(8, dtype=torch.float32, device=DEV)
    _lib.call("xb_ppg_aux_gauss_loss_fwd_bwd", *[_lib.ptr(t) for t in ins], B, D, B if B_total is None else B_total,
              float(kl_beta), _lib.ptr(dmu), _lib.ptr(dls), _lib.ptr(dv), _lib.ptr(da), _lib.ptr(st),
              _lib.ptr(_lib.scratch(DEV)))
    return [t.cpu().numpy() for t in (dmu, dls, dv, da, st)]


def _close_stats(got, want):
    np.testing.assert_allclose(got[:5], want[:5], rtol=2e-5, atol=1e-6)


# ====================================================================================================== kernels
@pytest.mark.parametrize("B", [1, 255, 256, 257])
@pytest.mark.parametrize("A", [1, 2, 17, 64])
def test_cat_kernel_matches_float64(B, A):
    rng = np.random.default_rng(B * 100 + A)
    z, o, v, aux, ret = cat_batch(rng, B, A)
    kl_beta = 0.7
    dz, dv, da, st = _cat_launch(z, o, v, aux, ret, kl_beta)
    rdz, rdv, rda, rst, _ = cat_aux_ref(z, o, v, aux, ret, kl_beta)
    np.testing.assert_allclose(dz, rdz, rtol=1e-3, atol=2e-6 * kl_beta / B)
    np.testing.assert_allclose(dv, rdv, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(da, rda, rtol=1e-6, atol=1e-9)
    _close_stats(st, rst)
    if A > 1 and B > 1:
        assert np.isinf(st[1]) and np.isinf(st[3])             # a q = 0 term under p > 0: the KL is +inf, as torch
        assert np.isfinite(dz).all()                          # ... and passes no gradient


@pytest.mark.parametrize("A", [17, 64])
def test_cat_kernel_large_batch_and_bit_identity(A):
    rng = np.random.default_rng(9)
    z, o, v, aux, ret = cat_batch(rng, BIG, A, zeros=False)
    first = _cat_launch(z, o, v, aux, ret, 1.0)
    rdz, rdv, rda, rst, _ = cat_aux_ref(z, o, v, aux, ret, 1.0)
    np.testing.assert_allclose(first[0], rdz, rtol=1e-3, atol=2e-6 / BIG)
    _close_stats(first[3], rst)
    for _ in range(2):
        again = _cat_launch(z, o, v, aux, ret, 1.0)
        for a, b in zip(first, again):
            np.testing.assert_array_equal(a, b)


def test_cat_kernel_zero_probability_and_nan_rules():
    """-inf logits on either side give autograd's NaN row (0 * inf); a NaN input propagates; finite-underflow zeros do
    not; new == old gives a KL of exactly 0."""
    rng = np.random.default_rng(4)
    z, o, v, aux, ret = cat_batch(rng, 8, 5, zeros=False)
    z[0, 1] = -np.inf                           # p = 0 from -inf
    o[1, 2] = -np.inf                           # q = 0 from -inf
    z[2, 3] = np.nan
    o[3] = z[3]                                 # new == old
    z[4, 0] -= 1e4                              # p = 0, finite
    dz, _, _, st = _cat_launch(z, o, v, aux, ret, 1.0)
    rdz, _, _, _, kl = cat_aux_ref(z, o, v, aux, ret, 1.0)
    np.testing.assert_allclose(dz, rdz, rtol=1e-3, atol=1e-6)
    assert np.isnan(dz[0]).all() and np.isnan(dz[1]).all() and np.isnan(dz[2]).all()
    assert np.isfinite(dz[3:]).all()
    assert np.isnan(st[1])
    _, _, _, st3 = _cat_launch(z[3:4], o[3:4], v[3:4], aux[3:4], ret[3:4], 1.0)
    assert st3[1] == 0.0


def test_cat_kernel_critic_only_form():
    rng = np.random.default_rng(2)
    _, _, v, _, ret = cat_batch(rng, 300, 2)
    dz, dv, da, st = _cat_launch(None, None, v, None, ret, 1.0)
    _, rdv, _, rst, _ = cat_aux_ref(None, None, v, None, ret, 1.0)
    np.testing.assert_allclose(dv, rdv, rtol=1e-6)
    _close_stats(st, rst)
    assert st[0] == 0 and st[1] == 0 and st[3] == st[2]
    from xuance_b200 import _lib                # the critic-only form takes no A: an A over the limit is not an error
    vd, rd = _d(v), _d(ret)
    dv65, st65 = torch.empty_like(vd), torch.empty(8, dtype=torch.float32, device=DEV)
    _lib.call("xb_ppg_aux_loss_fwd_bwd", None, None, _lib.ptr(vd), None, _lib.ptr(rd), len(v), 65, len(v), 1.0, None,
              _lib.ptr(dv65), None, _lib.ptr(st65), _lib.ptr(_lib.scratch(DEV)))
    np.testing.assert_array_equal(dv65.cpu().numpy(), dv)
    np.testing.assert_array_equal(st65.cpu().numpy(), st)


@pytest.mark.parametrize("G", [2, 3, 8])
def test_shards_sum_to_the_full_batch(G):
    rng = np.random.default_rng(G)
    B = 257
    z, o, v, aux, ret = cat_batch(rng, B, 6, zeros=False)
    full = _cat_launch(z, o, v, aux, ret, 0.5)
    mu, ls, omu, ols, gv, gaux, gret = gauss_batch(rng, B, 3)
    gfull = _gauss_launch(mu, ls, omu, ols, gv, gaux, gret, 0.5)
    parts, gparts = [], []
    for sl in np.array_split(np.arange(B), G):
        parts.append(_cat_launch(z[sl], o[sl], v[sl], aux[sl], ret[sl], 0.5, B_total=B))
        gparts.append(_gauss_launch(mu[sl], ls, omu[sl], ols, gv[sl], gaux[sl], gret[sl], 0.5, B_total=B))
    for i in range(3):                          # per-row outputs: the shards' rows are the full launch's, bit for bit
        np.testing.assert_array_equal(np.concatenate([p[i] for p in parts]), full[i])
    np.testing.assert_allclose(sum(p[3] for p in parts)[:3], full[3][:3], rtol=1e-6)
    for i in (0, 2, 3):
        np.testing.assert_array_equal(np.concatenate([p[i] for p in gparts]), gfull[i])
    np.testing.assert_allclose(sum(p[1] for p in gparts), gfull[1], rtol=1e-6)
    np.testing.assert_allclose(sum(p[4] for p in gparts)[:3], gfull[4][:3], rtol=1e-6)


@pytest.mark.parametrize("B", [1, 255, 256, 257])
@pytest.mark.parametrize("D", [1, 3, 6, 17, 64])
def test_gauss_kernel_matches_float64(B, D):
    rng = np.random.default_rng(B * 10 + D)
    args = gauss_batch(rng, B, D)
    got = _gauss_launch(*args, 0.9)
    want = gauss_aux_ref(*args, 0.9)
    np.testing.assert_allclose(got[0], want[0], rtol=1e-4, atol=1e-7 / (B * D))
    np.testing.assert_allclose(got[1], want[1], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(got[2], want[2], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(got[3], want[3], rtol=1e-6, atol=1e-9)
    _close_stats(got[4], want[4])


@pytest.mark.parametrize("D", [3, 64])
def test_gauss_kernel_large_batch_nan_and_bit_identity(D):
    rng = np.random.default_rng(11)
    args = list(gauss_batch(rng, BIG, D))
    first = _gauss_launch(*args, 1.0)
    want = gauss_aux_ref(*args, 1.0)
    np.testing.assert_allclose(first[0], want[0], rtol=1e-4, atol=1e-7 / (BIG * D))
    # a column whose scales nearly agree forms (h - h / vr) by cancellation in float32: tolerance on the scale there
    np.testing.assert_allclose(first[1], want[1], rtol=1e-4, atol=1e-6 * np.abs(want[1]).max())
    _close_stats(first[4], want[4])
    again = _gauss_launch(*args, 1.0)
    for a, b in zip(first, again):
        np.testing.assert_array_equal(a, b)
    args[0] = args[0][:9].copy()
    args[0][2, 1] = np.nan
    args[2:] = [args[2][:9], args[3], args[4][:9], args[5][:9], args[6][:9]]
    got = _gauss_launch(*args, 1.0)
    assert np.isnan(got[0][2, 1]) and np.isfinite(np.delete(got[0].ravel(), 2 * D + 1)).all()
    assert np.isfinite(got[1]).all() and np.isnan(got[4][1])       # as autograd: the scale gradient skips mu


# ====================================================================================================== learner
OBS, HORIZON, N_ENVS = 4, 16, 4


def _agent(discrete, **over):
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    env_id = "CartPole-v1" if discrete else "Pendulum-v1"
    kw = dict(device=DEV, parallels=N_ENVS, horizon_size=HORIZON, n_minibatch=2, running_steps=HORIZON * N_ENVS * 8,
              use_grad_clip=True, grad_clip_norm=0.5, model_dir="/tmp/xb_models/ppg_unit")
    kw.update(over)
    cfg = get_arguments("ppg", "classic_control", env_id, parser_args=Namespace(**kw))
    torch.manual_seed(0)
    act = Discrete(3) if discrete else Box(-1, 1, (2,), np.float32)
    return REGISTRY_Agents["PPG"](cfg, None, Box(-10, 10, (OBS,), np.float32), act)


def _fill(agent, seed=0):
    rng = np.random.default_rng(seed)
    mem = agent.memory
    gaussian = agent._gaussian_policy
    for _ in range(HORIZON):
        acts = rng.normal(size=(N_ENVS, 2)).astype(np.float32) if gaussian else rng.integers(0, 3, N_ENVS)
        mem.store(rng.normal(size=(N_ENVS, OBS)).astype(np.float32), acts, rng.normal(size=N_ENVS).astype(np.float32),
                  rng.normal(size=N_ENVS).astype(np.float32), rng.random(N_ENVS) < 0.1,
                  {"old_logp": (rng.normal(size=N_ENVS) * 0.3 - 1.0).astype(np.float32)})
    for i in range(N_ENVS):
        mem.finish_path(0.2, i)


def _oracle(agent):
    cfg, lrn = agent.config, agent.learner
    model = copy.deepcopy(agent.model)
    return PPGOracle(model, cfg.learning_rate, cfg.ent_coef, cfg.clip_range, cfg.kl_beta, cfg.use_grad_clip,
                     cfg.grad_clip_norm, lrn.end_factor_lr_decay, lrn.total_iters)


def _cpu(s):
    return {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in s.items()}


def _run_cycle(agent, orc, seed=1):
    """A full cycle with fixed minibatches: 2 x policy, 2 x critic, relabel, 2 x auxiliary.  Yields after each phase."""
    rng = np.random.default_rng(seed)
    mem, lrn = agent.memory, agent.learner
    gaussian = agent._gaussian_policy
    idxs = [rng.permutation(N_ENVS * HORIZON)[: N_ENVS * HORIZON // 2] for _ in range(2)]
    infos = {}
    for phase in ("actor", "critic", "aux"):
        if phase == "aux":
            agent._relabel()
            obs_all = mem.observations.reshape(-1, OBS).clone() if orc else None
            old_all = orc.relabel(obs_all) if orc else None
        for n, idx in enumerate(idxs):
            s = mem.sample(torch.as_tensor(idx, device=DEV))
            sync = n == len(idxs) - 1
            if phase == "actor":
                got = lrn.update_actor(sync=sync, **s)
                want = orc and orc.update_actor(s["obs"], s["actions"] if gaussian else s["actions"].long(),
                                                s["advantages"], s["aux_batch"]["old_logp"])
            elif phase == "critic":
                got = lrn.update_critic(sync=sync, **s)
                want = orc and orc.update_critic(s["obs"], s["returns"])
            else:
                got = lrn.update_auxiliary_critic(sync=sync, **s)
                old = None if orc is None else (old_all[0][idx], old_all[1]) if gaussian else (old_all[0][idx],)
                want = orc and orc.update_auxiliary_critic(s["obs"], s["returns"], old)
            if sync:
                infos[phase] = (got, want)
        yield phase, infos[phase]


def _assert_params_close(agent, orc, rtol=2e-4, atol=2e-5):
    for (k, a), (_, b) in zip(agent.model.state_dict().items(), orc.model.state_dict().items()):
        np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=rtol, atol=atol, err_msg=k)


def _steps(opt):
    sd = opt.state_dict()
    return {i: float(st["step"]) for i, st in sd["state"].items()}


@pytest.mark.parametrize("discrete", [True, False])
def test_learner_matches_oracle_phase_by_phase(discrete):
    torch.backends.cuda.matmul.allow_tf32 = False
    agent = _agent(discrete)
    _fill(agent)
    orc = _oracle(agent)
    keys = {"actor": {"actor-loss", "entropy", "learning_rate", "clip_ratio"}, "critic": {"critic-loss"},
            "aux": {"aux-loss", "kl-loss", "value-loss", "loss"}}
    for phase, (got, want) in _run_cycle(agent, orc):
        assert set(got) == keys[phase] == set(want)
        for k in got:
            assert got[k] == pytest.approx(want[k], rel=2e-4, abs=2e-5), (phase, k)
        _assert_params_close(agent, orc)
        assert _steps(agent.learner.optimizer) == _steps(orc.optimizer), phase
    # Adam moments too, parameter by parameter
    ours = agent.learner.optimizer.state_dict()["state"]
    theirs = orc.optimizer.state_dict()["state"]
    for i in theirs:
        for m in ("exp_avg", "exp_avg_sq"):
            np.testing.assert_allclose(ours[i][m].cpu().numpy(), theirs[i][m].cpu().numpy(), rtol=2e-3, atol=1e-7)


@pytest.mark.parametrize("discrete", [True, False])
def test_untouched_groups_stay_untouched(discrete):
    agent = _agent(discrete)
    _fill(agent)
    opt = agent.learner.optimizer
    groups = {"actor": agent.model.actor, "critic": agent.model.critic, "aux": agent.model.aux_critic}

    def snap():
        out = {}
        for g, mod in groups.items():
            a, b = opt.bounds[["actor", "critic", "aux"].index(g)]
            out[g] = (opt.bucket.flat[a:b].clone(), opt.exp_avg[a:b].clone(), opt.exp_avg_sq[a:b].clone())
        return out
    n_actor = len(list(agent.model.actor.parameters()))
    n_critic = len(list(agent.model.critic.parameters()))
    before = snap()
    assert opt.state_dict()["state"] == {}
    touched = {"actor": {"actor"}, "critic": {"actor", "critic"}, "aux": {"actor", "critic", "aux"}}
    for phase, _ in _run_cycle(agent, None):
        after = snap()
        for g in groups:
            same = all(torch.equal(x, y) for x, y in zip(before[g], after[g]))
            moved = g in (("actor",) if phase == "actor" else ("critic",) if phase == "critic" else groups)
            assert same != moved, (phase, g)
        before = after
        steps = _steps(opt)
        want = {"actor": {"actor": 2, "critic": 0, "aux": 0}, "critic": {"actor": 2, "critic": 2, "aux": 0},
                "aux": {"actor": 4, "critic": 4, "aux": 2}}[phase]
        for i in range(n_actor):
            assert steps.get(i, 0) == want["actor"]
        for i in range(n_actor, n_actor + n_critic):
            assert steps.get(i, 0) == want["critic"]
        assert all(steps.get(i, 0) == want["aux"] for i in range(n_actor + n_critic, len(list(agent.model.parameters()))))
        assert {g for g in groups if any(steps.get(i, 0) for i in _ids(agent, g))} == touched[phase]


def _ids(agent, g):
    n_a = len(list(agent.model.actor.parameters()))
    n_c = len(list(agent.model.critic.parameters()))
    n = len(list(agent.model.parameters()))
    return {"actor": range(0, n_a), "critic": range(n_a, n_a + n_c), "aux": range(n_a + n_c, n)}[g]


@pytest.mark.parametrize("discrete", [True, False])
def test_graphed_cycle_is_bit_equal_to_eager(discrete):
    torch.backends.cuda.matmul.allow_tf32 = False
    results = []
    for graph in (False, True):
        agent = _agent(discrete, use_cuda_graph=graph)
        _fill(agent)
        infos = [info for _, info in _run_cycle(agent, None)]
        if graph:
            assert agent.learner._graphs
        results.append(([t.clone() for t in agent.model.state_dict().values()], agent.learner.optimizer.exp_avg.clone(),
                        [i[0] for i in infos]))
    for a, b in zip(results[0][0], results[1][0]):
        assert torch.equal(a, b)
    assert torch.equal(results[0][1], results[1][1])
    assert results[0][2] == results[1][2]


def test_agent_train_epochs_runs_the_three_phases():
    agent = _agent(True)
    _fill(agent)
    np.random.seed(3)
    info = agent.train_epochs(agent.n_epochs)
    assert {"actor-loss", "entropy", "learning_rate", "clip_ratio", "critic-loss", "aux-loss", "kl-loss", "value-loss",
            "loss"} == set(info)
    steps = set(_steps(agent.learner.optimizer).values())
    cfg = agent.config
    per = agent.n_minibatch
    assert steps == {float((cfg.policy_nepoch + cfg.aux_nepoch) * per), float((cfg.value_nepoch + cfg.aux_nepoch) * per),
                     float(cfg.aux_nepoch * per)}
    assert agent.learner.scheduler.last_epoch == cfg.policy_nepoch * per


@pytest.mark.parametrize("kind,mb,clip", [(k, m, c) for k in ("cat", "gauss") for m in (1, 2) for c in (0, 1)])
@pytest.mark.parametrize("graph", [False, True])
def test_learner_matches_reference_fixture(kind, mb, clip, graph):
    """PPG_Learner replays the reference's full cycle (tests/golden/ppg_update.npz): the reference's minibatches, the
    relabel through this model's actor between the critic and the auxiliary phases, and after every phase the
    reference's infos, parameters and per-parameter Adam state (step exact; no state for a group never stepped)."""
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import PPG_Learner
    from xuance_b200.torch.rl_models import CategoricalDistribution, DiagGaussianDistribution
    from oracle_ppg import build_fixture_model
    from ppg_refs import FIX_INFO_KEYS, fix_learner_config
    torch.backends.cuda.matmul.allow_tf32 = False
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ppg_update.npz"))
    pre = f"{kind}/mb{mb}/clip{clip}/"
    model = build_fixture_model(kind, DEV)
    model.load_state_dict({k[len(pre + "init/"):]: torch.from_numpy(g[k]) for k in g.files
                           if k.startswith(pre + "init/")}, strict=True)
    cfg = Namespace(device=DEV, distributed_training=False, model_dir="/tmp/xb_models/ppg_fixture",
                    use_cuda_graph=graph, **fix_learner_config(mb, clip))
    lrn = PPG_Learner(cfg, model, BaseCallback())
    assert lrn.total_iters == int(g[pre + "total_iters"])
    t = lambda k: _d(g[pre + "in/" + k])
    obs, act, adv, ret, old_logp = t("obs"), t("actions"), t("advantages"), t("returns"), t("old_logp")
    names = [n for n, _ in model.named_parameters()]
    for phase in ("actor", "critic", "aux"):
        if phase == "aux":
            with torch.no_grad():
                if kind == "gauss":
                    mu, log_std = model.mu_log_std(obs)
                    mu, log_std = mu.clone(), log_std.detach().clone()
                else:
                    logits = model.logits(obs).clone()
        idxs = g[f"{pre}idx/{phase}"]
        for n, idx in enumerate(idxs):
            i = torch.as_tensor(idx, device=DEV)
            s = {"obs": obs[i], "actions": act[i], "advantages": adv[i], "returns": ret[i]}
            sync = n == len(idxs) - 1
            if phase == "actor":
                info = lrn.update_actor(sync=sync, aux_batch={"old_logp": old_logp[i]}, **s)
            elif phase == "critic":
                info = lrn.update_critic(sync=sync, aux_batch={}, **s)
            else:
                if kind == "gauss":
                    d = DiagGaussianDistribution(mu.shape[1])
                    d.set_param(mu[i], log_std.exp().expand(len(idx), -1))
                    aux = {"old_dist": d, "old_dist_log_std": log_std}
                else:
                    d = CategoricalDistribution(logits.shape[1])
                    d.set_param(logits=logits[i])
                    aux = {"old_dist": d}
                info = lrn.update_auxiliary_critic(sync=sync, aux_batch=aux, **s)
            if sync:
                np.testing.assert_allclose([info[k] for k in FIX_INFO_KEYS[phase]], g[f"{pre}info/{phase}"][n],
                                           rtol=1e-4, atol=1e-6, err_msg=phase)
        after = f"{pre}after/{phase}/"
        for k, v in model.state_dict().items():
            np.testing.assert_allclose(v.cpu().numpy(), g[after + k], rtol=1e-4, atol=1e-5, err_msg=f"{phase} {k}")
        state = lrn.optimizer.state_dict()["state"]
        assert {names[i] for i in state} == {k[len(after + "adam/"):].split("/")[0] for k in g.files
                                             if k.startswith(after + "adam/")}, phase
        for i, st in state.items():
            assert float(st["step"]) == float(g[f"{after}adam/{names[i]}/step"]), (phase, names[i])
            for m in ("exp_avg", "exp_avg_sq"):       # entries near 0 are sums that cancel: tolerance on the scale
                want = g[f"{after}adam/{names[i]}/{m}"]
                np.testing.assert_allclose(st[m].cpu().numpy(), want, rtol=2e-3, atol=1e-4 * np.abs(want).max(),
                                           err_msg=f"{phase} {names[i]} {m}")


# ====================================================================================================== buffer
@pytest.mark.parametrize("discrete", [True, False])
def test_buffer_old_dist_gather_and_checkpoint(discrete):
    agent = _agent(discrete)
    _fill(agent)
    agent._relabel()
    mem = agent.memory
    rows = mem.aux_rows["old_dist"]
    idx = torch.as_tensor(np.random.default_rng(0).permutation(N_ENVS * HORIZON)[:20], device=DEV)
    d = mem.sample(idx)["aux_batch"]["old_dist"]
    flat = rows.reshape(-1, rows.shape[-1])
    if discrete:
        want = torch.distributions.Categorical(logits=flat[idx]).logits
        assert torch.equal(d.logits, want)
    else:
        assert torch.equal(d.mu, flat[idx])
        assert torch.equal(d.std, mem.dist_log_std.exp().expand(20, 2))
        assert torch.equal(mem.dist_log_std, agent.model.actor.actor_head.log_std.detach())
        assert torch.equal(mem.sample(idx)["aux_batch"]["old_dist_log_std"], mem.dist_log_std)
    assert torch.equal(mem._gather_rows(rows, idx), flat[idx])
    sd = mem.state_dict()
    assert "_aux_rows_old_dist" in sd and torch.equal(sd["_aux_rows_old_dist"], rows.cpu())
    other = _agent(discrete)
    other.memory.load_state_dict(sd)
    assert torch.equal(other.memory.aux_rows["old_dist"], rows)
    if not discrete:
        assert torch.equal(other.memory.dist_log_std, mem.dist_log_std)


# ====================================================================================================== learning
def _learn(env_id, steps, device_rollout=False):
    from xuance_b200 import get_runner
    runner = get_runner("ppg", "classic_control", env_id,
                        parser_args=Namespace(device=DEV, running_steps=steps, device_rollout=device_rollout,
                                              model_dir="/tmp/xb_models/ppg_%s_%d" % (env_id, device_rollout)))
    agent = runner.agent
    before = float(np.mean(agent.test(test_episodes=10)))
    runner.run("train", running_steps=steps)
    assert {"actor-loss", "critic-loss", "aux-loss", "kl-loss"} <= set(agent.logged)
    after = float(np.mean(agent.test(test_episodes=10)))
    runner.finish()
    print("ppg %s device_rollout=%s before %.1f after %.1f" % (env_id, device_rollout, before, after))
    return before, after


# The shipped configs (10 envs x 256 steps per update cycle; 4 policy, 8 critic and 8 auxiliary epochs of one
# minibatch), seed 1.  Mean score of 10 stochastic test episodes before -> after training, measured on an
# H100 80GB HBM3 at its 700 W power limit:
#   CartPole-v1, 76800 steps (30 cycles): host 14.1 -> 500.0, device_rollout 14.1 -> 500.0  (a random policy: ~22)
#   Pendulum-v1, 128000 steps (50 cycles): host -1467.3 -> -1175.8 (+292); a second run -1467.3 -> -1186.5 (+281)
#   (a random policy: -1200 to -1500)
# The required CartPole score, 150, is far above random and far below the measured 500; the required Pendulum gain,
# 150, is about half the measured one (with one minibatch per epoch the reference's Pendulum settings learn slowly).
CARTPOLE_STEPS = 76800
PENDULUM_STEPS = 128000


@pytest.mark.parametrize("device_rollout", [False, True])
def test_ppg_cartpole_learns(device_rollout):
    before, after = _learn("CartPole-v1", CARTPOLE_STEPS, device_rollout)
    assert after > 150.0, (before, after)


def test_ppg_pendulum_learns():
    before, after = _learn("Pendulum-v1", PENDULUM_STEPS)
    assert after > before + 150.0, (before, after)

"""MAPPO on the device: K4M against its float64 restatement (every A tier, row counts around the block size and above
the grid-stride threshold, each switch, masked rows), sharded minibatches, determinism, the Σmask = 0 rule, the
ValueNorm update, the buffer's value-normalised GAE against the reference's loop, the learner against the torch-CPU
oracle and under a CUDA graph, and learning through REGISTRY_Agents["MAPPO"]."""
import copy
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
MAPPO_CONFIG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "xuance_b200", "configs",
                            "mappo", "sc2", "5m_vs_6m.yaml")   # the reference's configs/mappo/sc2/ layout
from mappo_refs import mappo_loss_ref, value_norm_update_f32, finish_path_ref, mean_std_f32  # noqa: E402
from oracle_mappo import MAPPOLearnerOracle  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _lib():
    from xuance_b200 import _lib
    _lib.load()
    return _lib


def _rows(rng, R, A):
    logits = rng.normal(0, 1.5, (R, A)).astype(np.float32)
    ld = (A + 3) // 4 * 4
    avail = np.zeros((R, ld), np.uint8)
    avail[:, :A] = rng.random((R, A)) > 0.3
    act = rng.integers(0, A, R)
    avail[np.arange(R), act] = 1
    avail[::7, :A] = 0
    avail[::7][np.arange(len(avail[::7])), act[::7]] = 1          # rows with a single available action
    f = lambda *a: rng.normal(*a).astype(np.float32)
    value = f(0, 2, R)
    return dict(logits=logits, avail=avail, actions=act.astype(np.float32), old_logp=f(-1.5, 0.6, R), adv=f(0, 1, R),
                value=value, old_value=(value + f(0, 0.1, R)).astype(np.float32), ret=f(0, 15, R),
                mask=(rng.random(R) > 0.2).astype(np.float32))


def _launch(d, vn, prep, R_total, clip, vclip, hdelta, masked, lo=0, hi=None):
    L = _lib()
    hi = len(d["actions"]) if hi is None else hi
    t = {k: torch.from_numpy(np.ascontiguousarray(v[lo:hi])).to(DEV) for k, v in d.items()}
    R, A = t["logits"].shape
    dl, dv = torch.empty_like(t["logits"]), torch.empty_like(t["value"])
    stats = torch.zeros(8, device=DEV)
    vn_t = None if vn is None else torch.tensor(vn, dtype=torch.float32, device=DEV)
    av = t["avail"] if masked else None
    L.call("xb_mappo_loss_fwd_bwd", L.ptr(t["logits"]), L.ptr(av), 0 if av is None else av.shape[1],
           L.ptr(t["actions"]), L.ptr(t["old_logp"]), L.ptr(t["adv"]), L.ptr(t["value"]), L.ptr(t["old_value"]),
           L.ptr(t["ret"]), L.ptr(t["mask"]), L.ptr(vn_t), L.ptr(prep), R, A, R_total, clip, vclip, hdelta, 1.0, 0.01,
           L.ptr(dl), L.ptr(dv), L.ptr(stats), L.ptr(L.scratch(DEV)))
    return dl.cpu().numpy(), dv.cpu().numpy(), stats.cpu().numpy()


def _prep(d):
    L = _lib()
    m, r = (torch.from_numpy(d[k]).to(DEV) for k in ("mask", "ret"))
    block = torch.zeros(4, dtype=torch.float64, device=DEV)
    L.call("xb_mappo_prepare", L.ptr(m), L.ptr(r), m.numel(), L.ptr(block), L.ptr(L.scratch(DEV)))
    return block


SWITCHES = [(0.2, 0.05, 10.0, True, True), (0.05, 0.0, 0.0, False, True), (0.2, 0.2, 0.0, True, False),
            (0.1, 0.0, 1.0, False, False)]


@pytest.mark.parametrize("A", [1, 5, 12, 19, 33, 64])
@pytest.mark.parametrize("R", [1, 255, 256, 257])
def test_k4m_matches_float64_reference(A, R):
    for k, (clip, vclip, hdelta, use_vn, masked) in enumerate(SWITCHES):
        rng = np.random.default_rng(1000 * A + R + k)
        d = _rows(rng, R, A)
        d["mask"][0] = 1.0
        vn = (0.7, 3.0) if use_vn else None
        prep = _prep(d)
        msum = float(prep[0])
        assert msum == float(d["mask"].sum())
        dl, dv, st = _launch(d, vn, prep, R, clip, vclip, hdelta, masked)
        rz, rv, rs = mappo_loss_ref(d["logits"], d["avail"] if masked else None, d["actions"], d["old_logp"], d["adv"],
                                    d["value"], d["old_value"], d["ret"], d["mask"], vn, msum, R, clip, vclip,
                                    hdelta, 1.0, 0.01)
        tol = lambda x: 2e-5 * max(1e-30, np.abs(x).max())
        np.testing.assert_allclose(dl, rz, rtol=1e-4, atol=tol(rz))
        np.testing.assert_allclose(dv, rv, rtol=1e-4, atol=tol(rv))
        np.testing.assert_allclose(st[:5], rs, rtol=1e-4, atol=1e-5 * max(1.0, np.abs(rs).max()))
        if masked:
            assert np.all(dl[d["avail"][:, :A] == 0] == 0.0)


def test_k4m_above_the_grid_stride_threshold():
    R, A = 2048 * 256 + 37, 5
    d = _rows(np.random.default_rng(5), R, A)
    prep = _prep(d)
    dl, dv, st = _launch(d, (0.1, 2.0), prep, R, 0.2, 0.05, 10.0, True)
    rz, rv, rs = mappo_loss_ref(d["logits"], d["avail"], d["actions"], d["old_logp"], d["adv"], d["value"],
                                d["old_value"], d["ret"], d["mask"], (0.1, 2.0), float(prep[0]), R, 0.2, 0.05, 10.0,
                                1.0, 0.01)
    np.testing.assert_allclose(dl, rz, rtol=1e-4, atol=2e-5 * np.abs(rz).max())
    np.testing.assert_allclose(dv, rv, rtol=1e-4, atol=2e-5 * np.abs(rv).max())
    np.testing.assert_allclose(st[:5], rs, rtol=1e-4)


@pytest.mark.parametrize("G", [2, 3, 8])
def test_k4m_shards_match_the_unsharded_launch(G):
    R, A = 1000, 12
    d = _rows(np.random.default_rng(G), R, A)
    prep = _prep(d)                                   # the all-reduced block every shard reads
    dl, dv, st = _launch(d, (0.3, 1.5), prep, R, 0.2, 0.05, 10.0, True)
    cuts = np.linspace(0, R, G + 1).astype(int)
    parts = [_launch(d, (0.3, 1.5), prep, R, 0.2, 0.05, 10.0, True, lo, hi) for lo, hi in zip(cuts[:-1], cuts[1:])]
    assert np.array_equal(np.concatenate([p[0] for p in parts]), dl)
    assert np.array_equal(np.concatenate([p[1] for p in parts]), dv)
    np.testing.assert_allclose(np.sum([p[2] for p in parts], axis=0), st, rtol=1e-6, atol=1e-7)


def test_k4m_statistics_are_deterministic_and_zero_mask_gives_nan():
    d = _rows(np.random.default_rng(9), 300000, 9)
    prep = _prep(d)
    a = _launch(d, None, prep, 300000, 0.2, 0.05, 10.0, True)
    b = _launch(d, None, prep, 300000, 0.2, 0.05, 10.0, True)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    d0 = _rows(np.random.default_rng(10), 64, 5)
    d0["mask"][:] = 0.0                               # the reference's 0/0: NaN losses and gradients, no guard
    dl, dv, st = _launch(d0, None, _prep(d0), 64, 0.2, 0.05, 10.0, False)
    assert np.isnan(st[:3]).all() and np.isnan(st[4]) and np.isfinite(st[3])
    assert np.isnan(dl).all() and np.isnan(dv).all()


def test_value_norm_update_matches_float32_order():
    from xuance_b200.torch.utils import ValueNorm
    vn = ValueNorm(1, device=DEV)
    state = (np.float32(0), np.float32(0), np.float32(0))
    rng = np.random.default_rng(0)
    for _ in range(5):
        r = rng.normal(4, 6, 777).astype(np.float32)
        vn.update(r)
        state, ms = value_norm_update_f32(*state, r, r.size)
        got = (vn.running_mean.item(), vn.running_mean_sq.item(), vn.debiasing_term.item())
        np.testing.assert_allclose(got, state, rtol=2e-7)
        np.testing.assert_allclose(vn.mean_std.cpu().numpy(), ms, rtol=5e-7)


@pytest.mark.parametrize("use_gae", [True, False])
@pytest.mark.parametrize("use_vn", [True, False])
def test_buffer_finish_path_and_sample_match_the_reference_loop(use_gae, use_vn):
    from xuance_b200.common import MARL_OnPolicyBuffer, Box, Discrete, AgentGrouping
    from xuance_b200.torch.utils import ValueNorm
    rng = np.random.default_rng(7)
    keys, n_envs, T, A = ["a0", "a1", "a2"], 2, 12, 7
    buf = MARL_OnPolicyBuffer(keys, None, {k: Box(-1, 1, (5,), np.float32) for k in keys},
                              {k: Discrete(A) for k in keys}, n_envs, n_envs * T, use_gae=use_gae, use_advnorm=True,
                              gamma=0.99, gae_lam=0.95, use_actions_mask=True,
                              avail_actions_shape={k: (A,) for k in keys}, device=DEV)
    grouping = AgentGrouping.shared(keys)
    vn = {"shared": ValueNorm(1, device=DEV)} if use_vn else None
    host = {f: np.zeros((n_envs, len(keys), T), np.float32) for f in ("rewards", "values", "terminals")}
    paths = []
    for t in range(T):
        step = {'obs': {k: rng.normal(size=(n_envs, 5)).astype(np.float32) for k in keys},
                'actions': {k: rng.integers(0, A, n_envs).astype(np.float32) for k in keys},
                'log_pi_old': {k: rng.normal(size=n_envs).astype(np.float32) for k in keys},
                'rewards': {k: rng.normal(size=n_envs).astype(np.float32) for k in keys},
                'values': {k: rng.normal(size=n_envs).astype(np.float32) for k in keys},
                'terminals': {k: np.array([t == 4, False]) for k in keys},
                'agent_mask': {k: np.ones(n_envs, bool) for k in keys},
                'avail_actions': {k: np.ones((n_envs, A), np.int64) for k in keys}}
        buf.store(**step)
        for f in host:
            for i, k in enumerate(keys):
                host[f][:, i, t] = step[f][k]
        if t == 4:                                    # env 0 ends a path early, with the state of that moment
            vnext = {k: 0.0 for k in keys}
            buf.finish_path(0, grouping, vnext, vn)
            paths.append((0, 0, 5, vnext, None if vn is None else mean_std_f32(
                *(x.item() for x in (vn["shared"].running_mean, vn["shared"].running_mean_sq,
                                     vn["shared"].debiasing_term)))))
            if vn is not None:
                vn["shared"].update(rng.normal(2, 3, 50).astype(np.float32))
    assert buf.full
    cur = None if vn is None else mean_std_f32(*(x.item() for x in (vn["shared"].running_mean,
                                                                      vn["shared"].running_mean_sq,
                                                                      vn["shared"].debiasing_term)))
    for e in range(n_envs):
        vnext = {k: float(rng.normal()) for k in keys}
        buf.finish_path(e, grouping, vnext, vn)
        paths.append((e, int(5 if e == 0 else 0), T, vnext, cur))
    ret = buf.field('returns').cpu().numpy().reshape(n_envs, len(keys), T)
    adv = buf.field('advantages').cpu().numpy().reshape(n_envs, len(keys), T)
    ref_adv = np.zeros_like(adv)
    for e, b, end, vnext, st in paths:
        for i, k in enumerate(keys):
            r, a = finish_path_ref(host['rewards'][e, i, b:end], host['values'][e, i, b:end],
                                   host['terminals'][e, i, b:end], np.float32(vnext[k]), use_gae, 0.99, 0.95, st)
            np.testing.assert_allclose(ret[e, i, b:end], r, rtol=1e-6, atol=1e-6)
            np.testing.assert_allclose(adv[e, i, b:end], a, rtol=1e-6, atol=1e-6)
            ref_adv[e, i, b:end] = a
    idx = rng.permutation(n_envs * T)[:10]
    s = buf.sample(idx)
    env, step = np.divmod(idx, T)
    for i, k in enumerate(keys):
        a = ref_adv[env, i, step]
        np.testing.assert_allclose(s['advantages'][k].cpu().numpy(), (a - a.mean()) / (a.std() + 1e-8), rtol=1e-4,
                                   atol=1e-5)
        np.testing.assert_array_equal(s['values'][k].cpu().numpy(), host['values'][env, i, step])


def _learner_cfg(**over):
    cfg = dict(agent="MAPPO", learner="MAPPO_Learner", device=DEV, learning_rate=7e-4, clip_range=0.05, vf_coef=1.0,
               ent_coef=0.01, use_value_clip=True, value_clip_range=0.05, use_value_norm=True, use_huber_loss=True,
               huber_delta=10.0, use_grad_clip=True, grad_clip_norm=10.0, use_linear_lr_decay=False,
               end_factor_lr_decay=0.5, running_steps=1000, buffer_size=32, n_epochs=1, n_minibatch=1,
               use_actions_mask=True, use_global_state=False, parallels=8, use_rnn=False, use_cuda_graph=False)
    cfg.update(over)
    return Namespace(**cfg)


def _model(device, obs_dim=12, A=7, keys=("a0", "a1", "a2")):
    from xuance_b200.common import AgentGrouping, Discrete
    from xuance_b200.torch.rl_models import (Basic_MLP, AgentFeatureEncoder, CategoricalActor,
                                             CentralizedStateValueCritic, MultiAgentActorCritic)
    g = AgentGrouping.shared(keys)
    torch.manual_seed(0)
    enc = lambda: AgentFeatureEncoder(Basic_MLP((obs_dim,), [32], activation=torch.nn.ReLU, device=device))
    actors = torch.nn.ModuleDict({"shared": CategoricalActor(enc(), [32], Discrete(A), activation=torch.nn.ReLU,
                                                             device=device)})
    critics = torch.nn.ModuleDict({"shared": CentralizedStateValueCritic(g, torch.nn.ModuleDict({"shared": enc()}),
                                                                         None, [32], activation=torch.nn.ReLU,
                                                                         device=device)})
    return g, MultiAgentActorCritic(g, actors, critics).to(device)


def _batch(rng, R, A=7, obs_dim=12, outside=False):
    avail = np.zeros((R, 8), np.uint8)
    avail[:, :A] = rng.random((R, A)) > 0.3
    act = rng.integers(0, A, R)
    avail[np.arange(R), act] = 1
    f = lambda *a: rng.normal(*a, R).astype(np.float32)
    old_logp = f(-2.0, 0.3) if not outside else np.where(rng.random(R) < 0.5, -8.0, 2.0).astype(np.float32)
    d = dict(obs=rng.normal(size=(R, obs_dim)).astype(np.float32), actions=act.astype(np.float32),
             log_pi_old=old_logp, advantages=f(0, 1), values=f(0, 0.5), returns=f(3, 20),
             agent_mask=(rng.random(R) > 0.15).astype(np.float32), avail_actions=avail)
    return d


def _as_sample(d):
    return {'_stacked': {k: torch.from_numpy(v).to(DEV) for k, v in d.items()}, 'batch_size': len(d['actions'])}


def test_learner_matches_the_torch_oracle():
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import MAPPO_Learner
    torch.backends.cuda.matmul.allow_tf32 = False
    g, model = _model(DEV)
    _, omodel = _model("cpu")
    omodel.load_state_dict({k: v.cpu() for k, v in model.state_dict().items()})
    cfg = _learner_cfg()
    learner = MAPPO_Learner(cfg, g, model, BaseCallback())
    oracle = MAPPOLearnerOracle(omodel, cfg)
    rng = np.random.default_rng(4)
    for it in range(3):
        d = _batch(rng, 96, outside=(it == 1))
        info = learner.update(_as_sample(d))
        t = {k: torch.from_numpy(v) for k, v in d.items()}
        oinfo = oracle.update(t['obs'], t['actions'], t['log_pi_old'], t['advantages'], t['values'], t['returns'],
                              t['agent_mask'], t['avail_actions'][:, :7])
        for k in ("actor_loss", "critic_loss", "entropy", "predict_value"):
            np.testing.assert_allclose(info["shared/" + k], oinfo[k], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(info["loss"], oinfo["loss"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(info["gradient_norm"], oinfo["gradient_norm"], rtol=1e-4)
        for (n, p), (_, q) in zip(model.state_dict().items(), omodel.state_dict().items()):
            np.testing.assert_allclose(p.cpu().numpy(), q.numpy(), rtol=1e-4, atol=2e-5, err_msg=n)
        vn, ovn = learner.value_normalizer["shared"], oracle.vn
        np.testing.assert_allclose(vn.running_mean.item(), ovn.running_mean.item(), rtol=1e-5)
        np.testing.assert_allclose(vn.debiasing_term.item(), ovn.debiasing_term.item(), rtol=1e-6)


def test_learner_cuda_graph_matches_eager():
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import MAPPO_Learner
    outs = []
    for graph in (False, True):
        g, model = _model(DEV)
        learner = MAPPO_Learner(_learner_cfg(use_cuda_graph=graph), g, model, BaseCallback())
        rng = np.random.default_rng(11)
        infos = [learner.update(_as_sample(_batch(rng, 128))) for _ in range(4)]
        outs.append(([p.detach().cpu().numpy() for p in model.parameters()], infos,
                     learner.value_normalizer["shared"].running_mean.item()))
    for a, b in zip(outs[0][0], outs[1][0]):
        assert np.array_equal(a, b)
    assert outs[0][1] == outs[1][1] and outs[0][2] == outs[1][2]


def test_mappo_learns_through_the_agent_registry():
    """REGISTRY_Agents["MAPPO"] on the cue-following SMAC-shaped env: the greedy team score rises well above chance
    (about 0.13 per step with ~7.7 available actions per agent; episodes of at most 20 steps)."""
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import REGISTRY_Agents
    cfg = get_arguments("mappo", "sc2", config_path=MAPPO_CONFIG)
    for k, v in dict(device=DEV, vectorize="Dummy_StarCraft2", parallels=8, buffer_size=256, running_steps=24000,
                     episode_limit=20, p_death=0.02, learning_rate=2e-3, clip_range=0.2, n_epochs=5,
                     model_dir="/tmp/xb200_mappo_models", log_dir="/tmp/xb200_mappo_logs").items():
        setattr(cfg, k, v)
    from xuance_b200.common import BaseCallback

    class Counting(BaseCallback):
        def __init__(self):
            self.calls = {}

        def _count(self, name):
            self.calls[name] = self.calls.get(name, 0) + 1
            return {}

        on_train_step = lambda self, *a, **k: self._count("on_train_step")
        on_train_step_end = lambda self, *a, **k: self._count("on_train_step_end")
        on_train_epochs_end = lambda self, *a, **k: self._count("on_train_epochs_end")
        on_train_episode_info = lambda self, *a, **k: self._count("on_train_episode_info")
    cb = Counting()
    envs = make_envs(cfg)
    agent = REGISTRY_Agents["MAPPO"](cfg, envs, callback=cb)
    before = float(np.mean(agent.test(16, test_envs=make_envs(cfg))))
    agent.train(cfg.running_steps // cfg.parallels)
    info = agent.logged
    after = float(np.mean(agent.test(32, test_envs=make_envs(cfg))))
    print("MAPPO learning: before %.3f after %.3f" % (before, after))
    assert np.isfinite(info.get("loss", np.nan)) and "shared/actor_loss" in info
    # one H100 80GB HBM3 run (700 W): before 3.37, after 14.51; the bar is set well below it
    assert after > before + 4.0 and after > 8.0, (before, after)
    steps = cfg.running_steps // cfg.parallels
    assert cb.calls["on_train_step"] == cb.calls["on_train_step_end"] == steps
    assert cb.calls["on_train_epochs_end"] == steps * cfg.parallels // cfg.buffer_size
    assert cb.calls["on_train_episode_info"] > 0
    agent.finish()


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mappo_update.npz")
GKEYS = [f"agent_{i}" for i in range(3)]


@pytest.mark.parametrize("case", ["gae1_vn0", "gae1_vn1", "gae0_vn0"])
def test_buffer_matches_reference_fixture(case):
    """store -> finish_path (a terminal path at t = 4, then the full buffer) -> sample with per-agent advantage
    normalisation, against the unmodified reference.  Float32 restatements of float64 steps (terminal paths) and the
    ValueNorm moments (fp64 sums here, float32 in torch) leave a few ulp."""
    from xuance_b200.common import MARL_OnPolicyBuffer, Box, Discrete, AgentGrouping
    from xuance_b200.torch.utils import ValueNorm
    from mappo_refs import mappo_buffer_steps
    g = np.load(GOLDEN)
    use_gae, use_vn = case.startswith("gae1"), case.endswith("vn1")
    rng = np.random.default_rng(5 + 2 * use_gae + use_vn)
    n_envs, T, A = 2, 12, 7
    buf = MARL_OnPolicyBuffer(GKEYS, None, {k: Box(-1, 1, (12,), np.float32) for k in GKEYS},
                              {k: Discrete(A) for k in GKEYS}, n_envs, n_envs * T, use_gae=use_gae, use_advnorm=True,
                              gamma=0.99, gae_lam=0.95, use_actions_mask=True,
                              avail_actions_shape={k: (A,) for k in GKEYS}, device=DEV)
    grouping = AgentGrouping.shared(GKEYS)
    vn = None
    if use_vn:
        vn = {"shared": ValueNorm(1, device=DEV)}
        vn["shared"].update(rng.normal(1.0, 4.0, (40, 1)).astype(np.float32))
    steps, nexts, vn_upd = mappo_buffer_steps(rng, GKEYS, n_envs, T, 12, A)
    for t, st in enumerate(steps):
        buf.store(**st)
        if t == 4:
            buf.finish_path(0, grouping, {k: 0.0 for k in GKEYS}, vn)
            if use_vn:
                vn["shared"].update(vn_upd)
    for e in range(n_envs):
        buf.finish_path(e, grouping, nexts[e], vn)
    if use_vn:
        st = [x.item() for x in (vn["shared"].running_mean, vn["shared"].running_mean_sq, vn["shared"].debiasing_term)]
        np.testing.assert_allclose(st, g[f"buffer/{case}/vn_state"], rtol=1e-6)
    for f in ("returns", "advantages"):
        got = buf.field(f).cpu().numpy().reshape(n_envs, 3, T).transpose(1, 0, 2)
        np.testing.assert_allclose(got, g[f"buffer/{case}/{f}"], rtol=1e-5, atol=1e-5)
    s = buf.sample(g[f"buffer/{case}/idx"])
    got = np.stack([s['advantages'][k].cpu().numpy() for k in GKEYS])
    np.testing.assert_allclose(got, g[f"buffer/{case}/sample_advantages"], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("graph", [False, True])
def test_learner_matches_reference_fixture(graph):
    from helpers import seeded_state_dict
    from mappo_refs import mappo_learner_batch
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import MAPPO_Learner
    torch.backends.cuda.matmul.allow_tf32 = False
    g = np.load(GOLDEN)
    grouping, model = _model(DEV, keys=tuple(GKEYS))
    model.load_state_dict(seeded_state_dict(model.state_dict(), 31))
    learner = MAPPO_Learner(_learner_cfg(huber_delta=1.0, use_cuda_graph=graph), grouping, model, BaseCallback())
    rng = np.random.default_rng(77)
    for it in range(3):
        b = mappo_learner_batch(rng, it, 32, GKEYS, 12, 7)
        d = {k: np.ascontiguousarray(np.asarray(v).reshape(96, *np.asarray(v).shape[2:])) for k, v in b.items()
             if k != 'batch_size'}
        d['agent_mask'] = d['agent_mask'].astype(np.float32)
        av = np.zeros((96, 8), np.uint8)
        av[:, :7] = d['avail_actions']
        d['avail_actions'] = av
        info = learner.update(_as_sample(d))
        got = [info["shared/" + k] for k in ("actor_loss", "critic_loss", "entropy", "predict_value")]
        got += [info["loss"], info["gradient_norm"], info["learning_rate"]]
        np.testing.assert_allclose(got, g["learner/infos"][it], rtol=2e-4, atol=2e-6)
        vn = learner.value_normalizer["shared"]
        np.testing.assert_allclose([vn.running_mean.item(), vn.running_mean_sq.item(), vn.debiasing_term.item()],
                                   g[f"learner/vn_state/{it}"], rtol=1e-6)
    for k, v in model.state_dict().items():
        np.testing.assert_allclose(v.cpu().numpy(), g[f"learner/final/{k}"], rtol=1e-4, atol=2e-5, err_msg=k)


def test_k4m_float32_tie_and_clip_boundary_rules():
    """torch.maximum tie with the clipped branch blocked (half of the unclipped gradient) and the value-clip boundary
    (inclusive: the full gradient), in the kernel's float32, exact in binary."""
    d = dict(logits=np.zeros((2, 3), np.float32), avail=np.ones((2, 4), np.uint8), actions=np.zeros(2, np.float32),
             old_logp=np.full(2, -np.log(3), np.float32), adv=np.zeros(2, np.float32),
             value=np.array([1.0, 0.25], np.float32), old_value=np.zeros(2, np.float32),
             ret=np.array([0.625, 1.0], np.float32), mask=np.ones(2, np.float32))
    _, dv, _ = _launch(d, None, _prep(d), 2, 0.2, 0.25, 0.0, False)
    assert dv[0] == np.float32(0.5 * 0.5 * 2 * 0.375) and dv[1] == np.float32(0.5 * 2 * (0.25 - 1.0))

"""GPU tests of recurrent MAPPO: MARL_OnPolicyBuffer_RNN against the reference's fixture (staging after every
finish_path, the ring, sample), the recurrent MAPPO_Learner against a torch-CPU oracle (nn.GRU on the CPU) eager and as a
CUDA graph, checkpoints, and REGISTRY_Agents["MAPPO"] from configs/mappo/sc2/3m.yaml learning on SyntheticSMACEnv."""
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from mappo_rnn_refs import scenario, KEYS, N_ENVS, N_AGENTS, T_MAX, SLOTS, OBS, STATE, A, SAMPLE  # noqa: E402
from oracle_mappo import MAPPOLearnerOracle  # noqa: E402
from oracle_mappo_rnn import RecurrentModelOracle  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mappo_rnn_buffer.npz")
FIELDS = ('actions', 'rewards', 'values', 'log_pi_old', 'terminals', 'agent_mask', 'returns', 'advantages')
EXACT = ('actions', 'rewards', 'values', 'log_pi_old', 'terminals', 'agent_mask')
# The GAE recursion is float64 in both (the reference through .item() / NumPy promotion, here K2's fp64 scan) with
# float32 stores; every case of the fixture agrees within this on an H100.
GAE_TOL = dict(rtol=1e-6, atol=1e-6)


def _buffer(use_gae):
    from xuance_b200.common import MARL_OnPolicyBuffer_RNN
    from xuance_b200.common.spaces import Box, Discrete
    return MARL_OnPolicyBuffer_RNN(KEYS, state_space=Box(-1, 1, (STATE,)), obs_space={k: Box(-1, 1, (OBS,)) for k in KEYS},
                                   act_space={k: Discrete(A) for k in KEYS}, n_envs=N_ENVS, buffer_size=SLOTS,
                                   max_episode_steps=T_MAX, use_gae=use_gae, use_advnorm=True, gamma=0.99, gae_lam=0.95,
                                   use_actions_mask=True, avail_actions_shape={k: (A,) for k in KEYS}, device=DEV)


def _check_staging(buf, g, pre):
    for f in FIELDS:
        dev = buf.field(f).cpu().numpy().reshape(N_ENVS, N_AGENTS, T_MAX)
        for i, k in enumerate(KEYS):
            ref = g[pre + f"{f}/{k}"].astype(np.float32)
            if f in EXACT:
                np.testing.assert_array_equal(dev[:, i], ref, err_msg=pre + f)
            else:
                np.testing.assert_allclose(dev[:, i], ref, err_msg=pre + f, **GAE_TOL)
    obs = buf._ep_obs.cpu().numpy().reshape(N_ENVS, N_AGENTS, T_MAX, OBS)
    for i, k in enumerate(KEYS):
        np.testing.assert_array_equal(obs[:, i], g[pre + f"obs/{k}"])
    np.testing.assert_array_equal(buf._ep_filled[0].cpu().numpy(), g[pre + "filled"].astype(np.float32))
    np.testing.assert_array_equal(buf._ep_state.cpu().numpy(), g[pre + "state"])


@pytest.mark.parametrize("use_gae,vn_on", [(True, False), (True, True), (False, False), (False, True)])
def test_buffer_matches_the_reference_fixture(use_gae, vn_on):
    from xuance_b200.common import AgentGrouping
    from xuance_b200.torch.utils import ValueNorm
    g = np.load(GOLDEN)
    case = f"gae{int(use_gae)}_vn{int(vn_on)}/"
    buf = _buffer(use_gae)
    vn = {"shared": ValueNorm(1, device=DEV)} if vn_on else None
    grouping = AgentGrouping.shared(KEYS)
    for j, op in enumerate(scenario()):
        if op[0] == "store":
            buf.store(**op[1])
        elif op[0] == "finish":
            _, e, i_step, vnext = op
            if vn_on:                  # the reference's ValueNorm state at this finish
                st = g[case + f"op{j}/vn"] if case + f"op{j}/vn" in g.files else None
                if st is None:         # the reference cannot run this case (non-GAE with a ValueNorm): see below
                    break
                v = vn["shared"]
                with torch.no_grad():
                    v.running_mean.fill_(float(st[0]))
                    v.running_mean_sq.fill_(float(st[1]))
                    v.debiasing_term.fill_(float(st[2]))
            buf.finish_path(i_env=e, i_step=i_step, agent_grouping=grouping, value_next=vnext, value_normalizer=vn)
            if case + "raises" not in g.files:
                _check_staging(buf, g, case + f"op{j}/staging/")
    if case + "raises" in g.files:
        # the reference raises a shape error here; this buffer computes what its GAE branch evidently intends:
        # returns by the discounted recursion, advantages = returns - denorm(values) (DESIGN §4)
        v = vn["shared"]
        mean, var = v.running_mean_var()
        T = 3                                    # env 0's first episode, in ring slot 0
        ring = lambda f: buf._scal[:N_AGENTS, FIELDS.index(f), :T].cpu().numpy().astype(np.float64)
        ret = np.zeros((N_AGENTS, T + 1))
        for t in range(T - 1, -1, -1):
            ret[:, t] = ring('rewards')[:, t] + (1 - ring('terminals')[:, t]) * 0.99 * ret[:, t + 1]
        den = ring('values') * np.sqrt(var.item()) + mean.item()
        np.testing.assert_allclose(ring('returns'), ret[:, :T], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(ring('advantages'), ret[:, :T] - den, rtol=1e-5, atol=1e-5)
        return
    for f in FIELDS:
        ring = buf._scal[:, FIELDS.index(f)].cpu().numpy().reshape(SLOTS, N_AGENTS, T_MAX)
        for i, k in enumerate(KEYS):
            ref = g[case + f"data/{f}/{k}"].astype(np.float32)
            if f in EXACT:
                np.testing.assert_array_equal(ring[:, i], ref, err_msg=f)
            else:
                np.testing.assert_allclose(ring[:, i], ref, err_msg=f, **GAE_TOL)
    np.testing.assert_array_equal(buf._filled.cpu().numpy(), g[case + "data/filled"].astype(np.float32))
    assert [buf.ptr, buf.size] == list(g[case + "ptr_size"]) and buf.full
    s = buf.sample(np.array(SAMPLE))
    assert [s["batch_size"], s["sequence_length"]] == list(g[case + "sample_meta"])
    for f in FIELDS + ('obs', 'avail_actions'):
        for k in KEYS:
            ref = g[case + f"sample/{f}/{k}"]
            got = s[f][k].cpu().numpy()
            if f in ('returns', 'advantages'):      # not normalised, although use_advnorm=True (as the reference)
                np.testing.assert_allclose(got, ref, **GAE_TOL)
            else:
                np.testing.assert_array_equal(got.astype(ref.dtype), ref, err_msg=f)
    np.testing.assert_array_equal(s["filled"].cpu().numpy(), g[case + "sample/filled"])
    np.testing.assert_array_equal(s["state"].cpu().numpy(), g[case + "sample/state"])
    # checkpoint round trip
    other = _buffer(use_gae)
    other.load_state_dict(buf.state_dict())
    s2 = other.sample(np.array(SAMPLE))
    for k, v in s["_stacked"].items():
        assert torch.equal(v, s2["_stacked"][k]), k


# ---------------------------------------------------------------- learner
def _model(obs_dim=OBS, n_actions=A, H=16):
    from xuance_b200.common import AgentGrouping, Discrete
    from xuance_b200.torch.rl_models import (Basic_RNN_K13, AgentFeatureEncoder, CategoricalActor,
                                             CentralizedStateValueCritic, MultiAgentActorCritic)
    g = AgentGrouping.shared(KEYS)
    torch.manual_seed(0)
    enc = lambda: AgentFeatureEncoder(Basic_RNN_K13((obs_dim,), normalize=nn.LayerNorm, initialize=nn.init.orthogonal_,
                                                    activation=nn.ReLU, device=DEV, fc_hidden_sizes=[24, 24],
                                                    recurrent_hidden_size=H))
    actors = nn.ModuleDict({"shared": CategoricalActor(enc(), [], Discrete(n_actions), initializer=nn.init.orthogonal_,
                                                       activation=nn.ReLU, device=DEV)})
    critics = nn.ModuleDict({"shared": CentralizedStateValueCritic(g, nn.ModuleDict({"shared": enc()}), None, [],
                                                                   initializer=nn.init.orthogonal_, activation=nn.ReLU,
                                                                   device=DEV)})
    return g, MultiAgentActorCritic(g, actors, critics, use_rnn=True).to(DEV)


def _learner_cfg(**over):
    cfg = dict(agent="MAPPO", learner="MAPPO_Learner", device=DEV, learning_rate=7e-4, clip_range=0.05, vf_coef=1.0,
               ent_coef=0.01, use_value_clip=True, value_clip_range=0.05, use_value_norm=True, use_huber_loss=True,
               huber_delta=1.0, use_grad_clip=True, grad_clip_norm=10.0, use_linear_lr_decay=False,
               end_factor_lr_decay=0.5, running_steps=1000, buffer_size=8, n_epochs=1, n_minibatch=1, episode_length=T_MAX,
               use_actions_mask=True, use_global_state=False, parallels=2, use_rnn=True, use_cuda_graph=False)
    cfg.update(over)
    return Namespace(**cfg)


def _batch(rng, B, T=12, outside=False):
    """B episodes x n agents of different lengths, dead agents, masked actions, returns on both Huber sides."""
    S = B * N_AGENTS
    lengths = np.tile(rng.integers(1, T + 1, B), N_AGENTS)
    filled = (np.arange(T)[None] < lengths[:, None]).astype(np.float32)
    avail = np.zeros((S, T, 4), np.uint8)
    avail[..., :A] = rng.random((S, T, A)) > 0.3
    act = rng.integers(0, A, (S, T))
    np.put_along_axis(avail, act[..., None], 1, axis=-1)
    f = lambda *a: rng.normal(*a, (S, T)).astype(np.float32)
    old = f(-1.4, 0.3) if not outside else np.where(rng.random((S, T)) < 0.5, -8.0, 2.0).astype(np.float32)
    return dict(obs=rng.normal(size=(S, T, OBS)).astype(np.float32), actions=act.astype(np.float32), log_pi_old=old,
                advantages=f(0, 1), values=f(0, 0.5), returns=f(1, 3), agent_mask=(rng.random((S, T)) > 0.15).astype(
                    np.float32), filled=filled, avail_actions=avail)


def _as_sample(d):
    return {'_stacked': {k: torch.from_numpy(v).to(DEV) for k, v in d.items()}, 'batch_size': len(d['actions']),
            'sequence_length': d['actions'].shape[1]}


@pytest.fixture
def strict_fp32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def test_recurrent_learner_matches_the_torch_oracle(strict_fp32):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import MAPPO_Learner
    g, model = _model()
    omodel = RecurrentModelOracle(model)
    cfg = _learner_cfg()
    learner = MAPPO_Learner(cfg, g, model, BaseCallback())
    oracle = MAPPOLearnerOracle(omodel, cfg)
    rng = np.random.default_rng(4)
    for it in range(3):
        d = _batch(rng, 6, outside=(it == 1))
        info = learner.update(_as_sample(d))
        t = {k: torch.from_numpy(v) for k, v in d.items()}
        fl = lambda k: t[k].reshape(-1)
        oinfo = oracle.update(t['obs'], fl('actions'), fl('log_pi_old'), fl('advantages'), fl('values'), fl('returns'),
                              fl('agent_mask') * fl('filled'), t['avail_actions'][..., :A].reshape(-1, A))
        for k in ("actor_loss", "critic_loss", "entropy", "predict_value"):
            np.testing.assert_allclose(info["shared/" + k], oinfo[k], rtol=1e-4, atol=1e-5, err_msg=k)
        np.testing.assert_allclose(info["loss"], oinfo["loss"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(info["gradient_norm"], oinfo["gradient_norm"], rtol=1e-4)
        osd = omodel.m.state_dict()
        for n, p in model.state_dict().items():
            np.testing.assert_allclose(p.cpu().numpy(), osd[n].numpy(), rtol=1e-4, atol=2e-5, err_msg=n)


def test_recurrent_learner_cuda_graph_matches_eager():
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import MAPPO_Learner
    outs = []
    for graph in (False, True):
        g, model = _model()
        learner = MAPPO_Learner(_learner_cfg(use_cuda_graph=graph), g, model, BaseCallback())
        rng = np.random.default_rng(11)
        infos = [learner.update(_as_sample(_batch(rng, 8))) for _ in range(4)]
        outs.append(([p.detach().cpu().numpy() for p in model.parameters()], infos,
                     learner.value_normalizer["shared"].running_mean.item()))
    for a, b in zip(outs[0][0], outs[1][0]):
        assert np.array_equal(a, b)
    assert outs[0][1] == outs[1][1] and outs[0][2] == outs[1][2]


def _cfg3m(**over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("mappo", "sc2", "3m")
    for k, v in dict(device=DEV, vectorize="Dummy_StarCraft2", model_dir="/tmp/xb200_mappo_rnn_models",
                     log_dir="/tmp/xb200_mappo_rnn_logs").items():
        setattr(cfg, k, v)
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def test_mappo_rnn_learns_through_the_agent_registry():
    """REGISTRY_Agents["MAPPO"] from configs/mappo/sc2/3m.yaml (use_rnn: True) on the cue-following SMAC-shaped env:
    the greedy team score rises well above its untrained value (one H100 80GB HBM3 run at 400 W: before 3.53, after
    12.95; the bar is set well below it)."""
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import REGISTRY_Agents
    cfg = _cfg3m(parallels=8, buffer_size=32, n_epochs=5, running_steps=16000, episode_limit=20, p_death=0.02,
                 learning_rate=2e-3)
    envs = make_envs(cfg)
    agent = REGISTRY_Agents["MAPPO"](cfg, envs)
    assert agent.use_rnn and type(agent.memory).__name__ == "MARL_OnPolicyBuffer_RNN"
    before = float(np.mean(agent.test(16, test_envs=make_envs(cfg))))
    agent.train(cfg.running_steps // cfg.parallels)
    info = agent.logged
    after = float(np.mean(agent.test(32, test_envs=make_envs(cfg))))
    print("recurrent MAPPO learning: before %.3f after %.3f" % (before, after))
    assert np.isfinite(info.get("loss", np.nan)) and "shared/actor_loss" in info
    assert after > before + 2.0, (before, after)
    # checkpoint round trip of the trained model into a fresh agent
    path = "/tmp/xb200_mappo_rnn_ckpt.pth"
    torch.save(agent.model.state_dict(), path)
    fresh = REGISTRY_Agents["MAPPO"](cfg, make_envs(cfg))
    fresh.model.load_state_dict(torch.load(path), strict=True)
    for (n, p), (_, q) in zip(agent.model.state_dict().items(), fresh.model.state_dict().items()):
        assert torch.equal(p, q), n
    agent.finish()
    fresh.finish()


def test_reference_5m_vs_6m_settings_run_with_use_rnn():
    """The reference's recurrent 5m_vs_6m settings (Basic_RNN, fc [64, 64, 64], GRU 64, LayerNorm) through
    get_arguments overrides: a short run trains and logs."""
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import REGISTRY_Agents
    cfg = get_arguments("mappo", "sc2", "5m_vs_6m")
    for k, v in dict(device=DEV, vectorize="Dummy_StarCraft2", use_rnn=True, representation="Basic_RNN", rnn="GRU",
                     N_recurrent_layers=1, fc_hidden_sizes=[64, 64, 64], recurrent_hidden_size=64, dropout=0,
                     parallels=4, buffer_size=4, n_epochs=2, running_steps=400, episode_limit=30,
                     model_dir="/tmp/xb200_mappo_rnn_models", log_dir="/tmp/xb200_mappo_rnn_logs").items():
        setattr(cfg, k, v)
    agent = REGISTRY_Agents["MAPPO"](cfg, make_envs(cfg))
    agent.train(cfg.running_steps // cfg.parallels)
    assert np.isfinite(agent.logged.get("loss", np.nan))
    agent.finish()

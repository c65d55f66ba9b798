"""Generate tests/golden/reference_live.pkl.gz by running the UNMODIFIED reference (agi-brain/xuance v1.4.4 @ 4f0b05b)
on the seeded inputs of tests/test_oracle_vs_reference.py, tests/test_dropin_reference.py and
tests/test_host_logic.py::test_running_mean_std_matches_reference, which compare the oracle with what is recorded here.

Needs a reference checkout (XB_REFERENCE_ROOT):   python tests/golden/make_reference_live.py
Models start from ``helpers.seeded_state_dict`` (loaded after the learner is built, as the oracle loads the reference
model's state in the tests), so no weights are stored; final parameters are stored as ``helpers.param_sample``.  The
recorded structures hold NumPy arrays and Python scalars only."""
import gzip
import inspect
import os
import pickle
import random
import sys
import textwrap
from argparse import Namespace
from copy import deepcopy
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.ref_loader import import_reference  # noqa: E402

import_reference()
from gymnasium.spaces import Box, Discrete  # noqa: E402
from helpers import synth_rollout, fill_buffers, qmix_episode_stream, seeded_state_dict, param_sample, digest  # noqa: E402

OUT = os.path.join(HERE, "reference_live.pkl.gz")


def plain(x):
    """NumPy / Python copy of a recorded structure (no reference or torch types)."""
    if isinstance(x, dict):
        return {k: plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(plain(v) for v in x)
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy().copy()
    if isinstance(x, np.ndarray):
        return x.copy()
    return x


def onpolicy():
    from xuance.common.memory_tools import DummyOnPolicyBuffer
    out = {}
    for seed, use_gae in [(0, True), (1, True), (2, False)]:
        rng = np.random.default_rng(seed)
        N, T = 5, 33
        ro = synth_rollout(rng, N, T, (3,), obs_dtype=np.float32, p_term=0.1)
        r = DummyOnPolicyBuffer(Box(-1, 1, (3,)), Discrete(4), {'old_logp': ()}, N, T, use_gae=use_gae)
        fill_buffers([r], ro, [(4, 1, np.float32(0.2)), (9, 3, 0.0), (20, 1, np.float32(-0.7))])
        idx = rng.permutation(N * T)[:50]
        s = r.sample(idx)
        out[seed] = dict(returns=r.returns.copy(), advantages=r.advantages.copy(),
                         sample={k: s[k].copy() for k in ('obs', 'actions', 'returns', 'values', 'advantages')})
    return out


def per():
    from xuance.common.memory_tools import PerOffPolicyBuffer
    out = {}
    for alpha in (0.5, 0.6):
        rng = np.random.default_rng(int(alpha * 10))
        N, S, B = 4, 64, 32
        r = PerOffPolicyBuffer(Box(-1, 1, (3,)), Discrete(4), None, N, N * S, B, alpha=alpha)
        r._max_priority = np.ones(N, np.float32)       # canonical float32 rule (oracle/replay.py docstring)
        events = []
        for t in range(100):
            st = (rng.normal(size=(N, 3)).astype(np.float32), rng.integers(0, 4, N), rng.normal(size=N).astype(np.float32),
                  rng.random(N) < 0.1, rng.normal(size=(N, 3)).astype(np.float32))
            r.store(*st)
            if t > 10 and t % 3 == 0:
                random.seed(t)
                s1 = r.sample(0.4)
                td = np.abs(rng.normal(size=B)).astype(np.float32)
                td[3] = 0
                r.update_priorities(s1['step_choices'], td)
                events.append(dict(t=t, step_choices=np.array(s1['step_choices']), weights=np.array(s1['weights']),
                                   sum=[digest(np.array(r._it_sum[i]._value, dtype=np.float64)) for i in range(N)],
                                   min=[digest(np.array(r._it_min[i]._value, dtype=np.float64)) for i in range(N)],
                                   max_priority=np.array(r._max_priority)))
        out[alpha] = events
    return out


def qmix_pair(n, obs_dim, A, S, T, lr_decay=0.5, seed=0):
    from xuance.common import BaseCallback, AgentGrouping
    from xuance.torch.rl_models.representations.rnn import Basic_RNN
    from xuance.torch.rl_models.representations.agent_feature import AgentFeatureEncoder
    from xuance.torch.rl_models.modules.identity_encoder import build_identity_encoder, IdentityFeatureFusion
    from xuance.torch.rl_models.critics.base_critics import DiscreteActionValueCritic
    from xuance.torch.rl_models.heads.q_mix_head import QMIX_Mixer
    from xuance.torch.rl_models.architectures.multi_agent.value_factorization import MixingQNetwork
    from xuance.torch.learners.multi_agent_rl.qmix_learner import QMIX_Learner
    keys = [f"agent_{i}" for i in range(n)]
    rep = Basic_RNN(input_shape=(obs_dim,), hidden_sizes=None, initialize=nn.init.orthogonal_, activation=nn.ReLU,
                    device='cpu', fc_hidden_sizes=[64], recurrent_hidden_size=64, N_recurrent_layers=1, dropout=0, rnn='GRU')
    enc = AgentFeatureEncoder(rep, build_identity_encoder(n, 'none', None, 'cpu'), IdentityFeatureFusion(64, 0, 'concat'))
    q = nn.ModuleDict({'shared': DiscreteActionValueCritic(enc, Discrete(A), [64], None, nn.init.orthogonal_, nn.ReLU, 'cpu')})
    grouping = AgentGrouping.shared(keys)
    model = MixingQNetwork(grouping, q, QMIX_Mixer(S, 32, 32, n, 'cpu'), use_rnn=True, device='cpu')
    cfg = Namespace(distributed_training=False, episode_length=T, use_grad_clip=False, grad_clip_norm=10, device='cpu',
                    model_dir='/tmp/x', running_steps=100000, parallels=4, use_parameter_sharing=True, use_rnn=True,
                    use_actions_mask=False, learning_rate=7e-4, sync_frequency=2, double_q=True, n_epochs=1,
                    start_training=0, gamma=0.99, end_factor_lr_decay=lr_decay)
    lrn = QMIX_Learner(cfg, grouping, model, BaseCallback())
    model.load_state_dict(seeded_state_dict(model.state_dict(), seed), strict=True)
    return keys, model, lrn


def qmix():
    from xuance.common.memory_tools_marl import MARL_OffPolicyBuffer_RNN
    n, obs_dim, A, S, T = 5, 72, 12, 98, 12
    keys, model, lrn = qmix_pair(n, obs_dim, A, S, T)
    init = {k: v.clone() for k, v in model.state_dict().items()}
    n_envs, C, Be = 3, 12, 6
    rb = MARL_OffPolicyBuffer_RNN(agent_keys=keys, state_space=Box(-1, 1, (S,)),
                                  obs_space={k: Box(-1, 1, (obs_dim,)) for k in keys},
                                  act_space={k: Discrete(A) for k in keys}, n_envs=n_envs, buffer_size=C,
                                  batch_size=Be, max_episode_steps=T, use_actions_mask=False)
    for ev in qmix_episode_stream(np.random.default_rng(0), keys, n_envs, T, obs_dim, A, S, 5):
        if ev[0] == 'store':
            rb.store(**ev[1])
        else:
            rb.finish_path(ev[1], **ev[2])
    data = {k: {a: digest(rb.data[k][a]) for a in keys} for k in ('obs', 'actions', 'rewards', 'terminals', 'agent_mask')}
    data['filled'], data['state'] = digest(rb.data['filled']), digest(rb.data['state'])
    upd = []
    for it in range(3):
        np.random.seed(it)
        i1 = lrn.update(rb.sample())
        upd.append(dict(loss_Q=float(i1['loss_Q']), predictQ=float(i1['predictQ']), learning_rate=i1['learning_rate']))
    sd = model.state_dict()
    moved = sorted(k for k in sd if k.startswith("individual_q_networks") and not torch.equal(sd[k], init[k]))
    assert not moved, moved          # the reference's agent networks receive no gradient with use_rnn=True
    return dict(total_iters=lrn.total_iters, data=data, ptr=rb.ptr, size=rb.size, updates=upd, final=param_sample(sd))


def sac():
    from xuance.common import BaseCallback
    from xuance.torch.rl_models.representations.mlp import Basic_Identical
    from xuance.torch.rl_models.actors.gaussian_actors import SAC_GaussianActor
    from xuance.torch.rl_models.critics.twin_critics import TwinActionValueCritic
    from xuance.torch.rl_models.architectures.single_agent.actor_critic import SoftActorCritic
    from xuance.torch.learners import SAC_Learner
    torch.manual_seed(0)
    obs_dim, act_dim, B = 17, 6, 64
    aspace = Box(-1, 1, (act_dim,), np.float32)
    rep = Basic_Identical((obs_dim,), device='cpu')
    actor = SAC_GaussianActor(rep, [256, 256], aspace, None, None, nn.LeakyReLU, nn.Tanh, 'cpu')
    critic = TwinActionValueCritic(deepcopy(rep), aspace, [256, 256], None, None, nn.LeakyReLU, 'cpu')
    model = SoftActorCritic(actor, critic)
    cfg = Namespace(distributed_training=False, episode_length=1000, use_grad_clip=False, grad_clip_norm=0.5, device='cpu',
                    model_dir='/tmp/x', running_steps=100000, parallels=4, start_training=0, training_frequency=1,
                    learning_rate_actor=1e-3, learning_rate_critic=1e-3, tau=0.005, gamma=0.99, alpha=0.2,
                    use_automatic_entropy_tuning=True, end_factor_lr_decay=0.7)
    lrn = SAC_Learner(cfg, model, BaseCallback())
    model.load_state_dict(seeded_state_dict(model.state_dict(), 1), strict=True)
    rng = np.random.default_rng(1)
    upd = []
    for it in range(3):
        s = {"obs": rng.normal(size=(B, obs_dim)).astype(np.float32),
             "actions": rng.uniform(-1, 1, size=(B, act_dim)).astype(np.float32),
             "obs_next": rng.normal(size=(B, obs_dim)).astype(np.float32),
             "rewards": rng.normal(size=B).astype(np.float32), "terminals": (rng.random(B) < 0.1).astype(np.float32)}
        torch.manual_seed(100 + it)
        i1 = lrn.update(**s)
        upd.append({k: float(i1[k]) for k in ("Qloss", "Ploss", "Qvalue", "alpha", "alpha_loss")})
    return dict(total_iters=lrn.total_iters, updates=upd, final=param_sample(model.state_dict()))


def siblings():
    from xuance.common import BaseCallback
    from xuance.torch.learners import A2C_Learner, PG_Learner, DDQN_Learner
    from xuance.torch.rl_models.representations import AC_CNN_Atari, Basic_CNN
    from xuance.torch.rl_models.heads import CategoricalActorHead, ValueHead
    from xuance.torch.rl_models.architectures.single_agent.actor_critic import SharedActorCritic
    from xuance.torch.rl_models.architectures.single_agent.deep_q_network import DeepQNetwork
    out = {}
    for kind in ("a2c", "pg", "ddqn"):
        torch.manual_seed(5)
        A, B = 5, 12
        cfg = Namespace(distributed_training=False, episode_length=1000, use_grad_clip=True, grad_clip_norm=0.5, device="cpu",
                        model_dir="/tmp/x", running_steps=4096 * 10, parallels=32, learning_rate=2.5e-4, end_factor_lr_decay=0.5,
                        horizon_size=128, n_epochs=4, n_minibatch=4, vf_coef=0.25, ent_coef=0.01, gamma=0.99, sync_frequency=2,
                        start_training=0, training_frequency=1)
        rng = np.random.default_rng(3)
        if kind == "ddqn":
            rep = Basic_CNN(input_shape=(84, 84, 4), kernels=[8, 4, 3], strides=[4, 2, 1], filters=[32, 64, 64],
                            activation=nn.ReLU, device="cpu")
            model = DeepQNetwork(rep, [512], Discrete(A), None, None, nn.ReLU, "cpu")
            lrn = DDQN_Learner(cfg, model, BaseCallback())
        else:
            rep = AC_CNN_Atari(input_shape=(84, 84, 4), kernels=[8, 4, 3], strides=[4, 2, 1], filters=[32, 64, 64],
                               activation=nn.ReLU, device="cpu", fc_hidden_sizes=[512])
            model = SharedActorCritic(rep, CategoricalActorHead(512, [], A, None, nn.init.orthogonal_, nn.ReLU, "cpu"),
                                      ValueHead(512, [], None, nn.init.orthogonal_, nn.ReLU, "cpu"))
            lrn = (A2C_Learner if kind == "a2c" else PG_Learner)(cfg, model, BaseCallback())
        model.load_state_dict(seeded_state_dict(model.state_dict(), 2), strict=True)
        upd = []
        for it in range(3):
            s = {"obs": rng.integers(0, 256, size=(B, 84, 84, 4), dtype=np.uint8).astype(np.float32),
                 "actions": rng.integers(0, A, size=B).astype(np.float32),
                 "returns": rng.normal(size=B).astype(np.float32), "advantages": rng.normal(size=B).astype(np.float32),
                 "aux_batch": {"old_logp": np.zeros(B, np.float32)},
                 "obs_next": rng.integers(0, 256, size=(B, 84, 84, 4), dtype=np.uint8).astype(np.float32),
                 "rewards": rng.normal(size=B).astype(np.float32), "terminals": (rng.random(B) < 0.2).astype(np.float32)}
            i1 = lrn.update(**s)
            upd.append({"Qloss": float(i1["Qloss"])} if kind == "ddqn" else
                       {"actor_loss": float(i1["actor-loss"]), "entropy": float(i1["entropy"])})
        out[kind] = dict(total_iters=lrn.total_iters, updates=upd, final=param_sample(model.state_dict()))
    return out


def ma_vec_env():
    from xuance.environment.utils.wrapper import XuanCeMultiAgentEnvWrapper as RefWrapper
    from xuance.environment.vector_envs.dummy.dummy_vec_maenv import DummyVecMultiAgentEnv as RefVec
    from xuance_b200.environment.ma_envs import SyntheticSMACEnv
    kw = dict(n_agents=3, obs_dim=16, state_dim=20, n_actions=5, episode_limit=7, p_death=0.1)
    n_envs = 3
    rv = RefVec([lambda env_seed=0: RefWrapper(SyntheticSMACEnv(seed=env_seed, **kw)) for _ in range(n_envs)], 11)
    rec = dict(num_envs=rv.num_envs, agents=list(rv.agents), num_agents=rv.num_agents,
               max_episode_steps=rv.max_episode_steps, state_shape=tuple(rv.state_space.shape))
    rec["reset"] = plain(rv.reset())
    rng = np.random.default_rng(2)
    steps = []
    for t in range(40):
        acts = [{a: int(rng.choice(np.flatnonzero(rv.buf_avail_actions[e][a]))) for a in rv.agents} for e in range(n_envs)]
        r = rv.step(acts)
        steps.append(dict(actions=acts, out=plain(tuple(r)), state=plain(rv.buf_state), avail=plain(rv.buf_avail_actions)))
    rv.close()
    rec["steps"] = steps
    return rec


def qmix_action_mask():
    from xuance.common.memory_tools_marl import MARL_OffPolicyBuffer_RNN
    from xuance.torch.learners.multi_agent_rl import iql_learner as iql
    n, obs_dim, A, S, T = 4, 24, 7, 30, 9
    keys, model, lrn = qmix_pair(n, obs_dim, A, S, T, seed=3)
    lrn.use_actions_mask = lrn.config.use_actions_mask = True
    n_envs, C, Be = 3, 12, 6
    rb = MARL_OffPolicyBuffer_RNN(agent_keys=keys, state_space=Box(-1, 1, (S,)),
                                  obs_space={k: Box(-1, 1, (obs_dim,)) for k in keys},
                                  act_space={k: Discrete(A) for k in keys}, n_envs=n_envs, buffer_size=C,
                                  batch_size=Be, max_episode_steps=T, use_actions_mask=True,
                                  avail_actions_shape={k: (A,) for k in keys})
    rng = np.random.default_rng(4)

    def avail(shape_prefix):
        a = rng.random(shape_prefix + (A,)) < 0.6
        a[..., 0] = True                                    # never an all-unavailable row
        return a
    for ev in qmix_episode_stream(np.random.default_rng(3), keys, n_envs, T, obs_dim, A, S, 5):
        if ev[0] == 'store':
            rb.store(avail_actions={k: avail((n_envs,)) for k in keys}, **ev[1])
        else:
            rb.finish_path(ev[1], avail_actions={k: avail(()) for k in keys}, **ev[2])
    np.random.seed(0)
    sample = rb.sample()
    snap = {k: v.clone() for k, v in model.state_dict().items()}
    try:                                                    # the reference as it is cannot run this configuration
        lrn.update(sample)
        raised = False
    except (RuntimeError, IndexError):
        raised = True
    assert raised
    model.load_state_dict(snap)
    lrn.iterations = 0
    # the same learner with the one slice of iql_learner.py:78 corrected, in memory only
    src = textwrap.dedent(inspect.getsource(iql.IQL_Learner._forward_transitions))
    bad = "batch.avail_actions.group(group)[:, 1:]"
    assert src.count(bad) == 1, "the reference's masked RNN branch changed - re-read iql_learner.py:60-81"
    scope = {}
    exec(compile(src.replace(bad, "batch.avail_actions.group(group)[:, :, 1:]"), "iql_learner.py (slice corrected)", "exec"),
         vars(iql), scope)
    iql.IQL_Learner._forward_transitions = scope["_forward_transitions"]
    samples, upd = [], []
    for it in range(3):
        np.random.seed(10 + it)
        s = rb.sample()
        samples.append(plain(s))
        i1 = lrn.update(s)
        upd.append(dict(loss_Q=float(i1['loss_Q']), predictQ=float(i1['predictQ'])))
    return dict(total_iters=lrn.total_iters, unpatched_raised=raised, samples=samples, updates=upd,
                final=param_sample(model.state_dict()))


def running_mean_std():
    from xuance.common.statistic_tools import RunningMeanStd as Ref
    rng = np.random.default_rng(1)
    a = Ref((3,))
    for _ in range(7):
        a.update(rng.normal(size=(8, 3)).astype(np.float32))
    return dict(mean=np.array(a.mean), var=np.array(a.var), count=a.count)


def train_epochs_calls():
    import xuance.torch.agents.core.on_policy as core

    class Recorder:
        def __init__(self):
            self.calls = []

        def sample(self, idx):
            self.calls.append(("sample", np.array(idx, copy=True)))
            return {"obs": idx[:1], "actions": idx[:1], "returns": idx[:1], "values": idx[:1], "advantages": idx[:1],
                    "aux_batch": {}, "batch_size": len(idx)}

        def update(self, **samples):
            self.calls.append(("update", tuple(sorted(samples))))
            return {"n": len(self.calls)}
    out = {}
    for buffer_size, batch_size, n_epochs in [(64, 16, 4), (60, 16, 3)]:
        rec = Recorder()
        agent = SimpleNamespace(buffer_size=buffer_size, batch_size=batch_size, memory=rec, learner=rec)
        np.random.seed(11)
        info = core.OnPolicyAgent.train_epochs(agent, n_epochs)
        out[(buffer_size, batch_size, n_epochs)] = dict(calls=rec.calls, info=plain(info))
    return out


if __name__ == "__main__":
    rec = dict(env="torch %s / numpy %s / reference 4f0b05b" % (torch.__version__, np.__version__),
               onpolicy=onpolicy(), per=per(), qmix=qmix(), sac=sac(), siblings=siblings(), ma_vec_env=ma_vec_env(),
               running_mean_std=running_mean_std(), train_epochs=train_epochs_calls(),
               qmix_action_mask=qmix_action_mask())   # last: it patches the reference's IQL learner in memory
    with gzip.open(OUT, "wb", compresslevel=9) as fh:
        pickle.dump(rec, fh, protocol=4)
    print(OUT, os.path.getsize(OUT), "bytes")

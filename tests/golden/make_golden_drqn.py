"""Generate tests/golden/drqn_update.npz by running the UNMODIFIED reference DRQN code (agi-brain/xuance v1.4.4) on CPU.

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_drqn.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs).

Learner (CASES below: LSTM at H = 128, LSTM at H = 17, GRU at H = 64): the reference's DeepRecurrentQNetwork on a
Basic_MLP representation built from torch.manual_seed(seed) - kept as the reference initialised it for FULL_CASE, loaded
with tests/oracle_drqn.py's seeded_state otherwise - and UPDATES DRQN_Learner.update calls with sync_frequency = 2 on
seeded samples whose window length changes between updates (L = lookup_length, then shorter).  Recorded: every sample,
every info dict, and for FULL_CASE in full (per-tensor sums and absolute sums for the others) the initial state_dict
(FULL_CASE only), the state_dict after the last update and the Adam moments after the last update.

Replay: the reference's RecurrentOffPolicyBuffer (n_envs = 2, n_size = 6) fed a seeded two-env stream of episodes,
some shorter than lookup_length, some truncated, more than n_size of them; SAMPLE_SEEDS seeded samples are recorded
after the stream.  Acting: ACT_STEPS seeded DRQN_Agent.get_actions steps (its source runs on a stand-in ``self`` holding
the model, the action space and n_envs) with a carried LSTM state, from seeded_state weights."""
import os
import sys
from collections import OrderedDict
from types import SimpleNamespace

import numpy as np
import torch

from make_golden import HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from oracle_drqn import seeded_state  # noqa: E402
from gymnasium.spaces import Discrete, Box  # noqa: E402
from xuance.common import BaseCallback, EpisodeBuffer, RecurrentOffPolicyBuffer  # noqa: E402
from xuance.torch.rl_models.representations import Basic_MLP  # noqa: E402
from xuance.torch.rl_models.architectures import DeepRecurrentQNetwork  # noqa: E402
from xuance.torch.learners.qlearning_family.drqn_learner import DRQN_Learner  # noqa: E402
from xuance.torch.agents.qlearning_family.drqn_agent import DRQN_Agent  # noqa: E402

# name, rnn, H, obs_dim, rep hidden, n_actions, B, lookup, windows per update, grad clip, seed
CASES = [("lstm128", "LSTM", 128, 4, 16, 2, 8, 50, (50, 50, 20, 20), False, 11),
         ("lstm17", "LSTM", 17, 5, 24, 3, 5, 12, (12, 7, 7, 12), True, 12),
         ("gru64", "GRU", 64, 4, 32, 2, 6, 10, (10, 6, 6, 10), True, 13)]
# the case whose initial weights are the reference's own initialisation (recorded in full); the others start from
# oracle_drqn.seeded_state(., seed), which the tests rebuild, and record digests only, to keep the fixture small
FULL_CASE = "lstm17"
UPDATES = 4
REPLAY = dict(n_envs=2, buffer_size=12, batch_size=5, episode_length=20, lookup_length=8, obs_dim=3, n_actions=3)
SAMPLE_SEEDS = (101, 102, 103)
ACT_STEPS = 6


def build_model(rnn, H, obs_dim, rep_hidden, n_actions, seed):
    torch.manual_seed(seed)
    rep = Basic_MLP(input_shape=(obs_dim,), hidden_sizes=[rep_hidden], normalize=None,
                    initialize=torch.nn.init.orthogonal_, activation=torch.nn.ReLU, device="cpu")
    return DeepRecurrentQNetwork(representation=rep, recurrent_hidden_size=H, recurrent_layer_N=1, dropout=0,
                                 action_space=Discrete(n_actions), rnn=rnn, initializer=torch.nn.init.orthogonal_,
                                 device="cpu")


def digest(v):
    """The per-tensor record of the digest-only cases: sum and absolute sum in float64."""
    v = np.asarray(v, np.float64)
    return np.array([v.sum(), np.abs(v).sum()])


def make_sample(rng, B, L, obs_dim, n_actions):
    return {"obs": rng.standard_normal((B, L + 1, obs_dim)).astype(np.float32),
            "actions": rng.integers(0, n_actions, (B, L)).astype(np.int64),
            "rewards": rng.standard_normal((B, L)).astype(np.float32),
            "terminals": (rng.random((B, L)) < 0.1).astype(np.float32), "batch_size": B}


def learner_config(clip, lookup):
    return _learner_cfg(learning_rate=1e-3, gamma=0.99, sync_frequency=2, use_grad_clip=clip, grad_clip_norm=0.5,
                        end_factor_lr_decay=0.5, running_steps=40, parallels=10, start_training=0,
                        training_frequency=1, lookup_length=lookup)


def golden_learner(out):
    for name, rnn, H, obs_dim, rep_hidden, A, B, lookup, windows, clip, seed in CASES:
        model = build_model(rnn, H, obs_dim, rep_hidden, A, seed)
        if name == FULL_CASE:
            for k, v in model.state_dict().items():
                out[f"{name}/init/{k}"] = v.numpy().copy()
        else:
            model.load_state_dict(seeded_state(model.state_dict(), seed), strict=True)
        learner = DRQN_Learner(learner_config(clip, lookup), model, BaseCallback())
        rng = np.random.default_rng(seed)
        for u, L in enumerate(windows):
            s = make_sample(rng, B, L, obs_dim, A)
            for k in ("obs", "actions", "rewards", "terminals"):
                out[f"{name}/u{u}/{k}"] = s[k]
            info = learner.update(**s)
            for k in ("Qloss", "learning_rate", "predictQ"):
                out[f"{name}/u{u}/info/{k}"] = np.float64(info[k])
        for k, v in model.state_dict().items():
            out[f"{name}/final/{k}"] = v.numpy().copy() if name == FULL_CASE else digest(v.numpy())
        named = OrderedDict(model.named_parameters())
        for pname, p in named.items():
            st = learner.optimizer.state.get(p)
            if not st:
                continue
            for m in ("exp_avg", "exp_avg_sq"):
                v = st[m].numpy()
                out[f"{name}/adam/{m}/{pname}"] = v.copy() if name == FULL_CASE else digest(v)


def replay_stream(seed=7):
    """A two-env stream: per step both envs add a transition; an env's episode ends at its drawn length, terminated
    or truncated.  Returns the per-step arrays and the (step, env) of every finished episode in storing order."""
    p = REPLAY
    rng = np.random.default_rng(seed)
    N, D = p["n_envs"], p["obs_dim"]
    lengths = [list(rng.integers(2, p["episode_length"] + 1, 12)) for _ in range(N)]
    for e in range(N):
        lengths[e][1] = 3                        # shorter than lookup_length
        lengths[e][2] = p["episode_length"]      # as long as possible
    init_obs = [rng.standard_normal(D).astype(np.float32) for _ in range(N)]
    steps, cursor, ep_idx, reset_obs = [], [0] * N, [0] * N, []
    n_steps = 60
    for t in range(n_steps):
        nxt = rng.standard_normal((N, D)).astype(np.float32)
        act = rng.integers(0, p["n_actions"], N).astype(np.int64)
        rew = rng.standard_normal(N).astype(np.float32)
        done = np.zeros(N, bool)
        term = np.zeros(N, bool)
        for e in range(N):
            cursor[e] += 1
            if cursor[e] == lengths[e][ep_idx[e]]:
                done[e] = True
                term[e] = rng.random() < 0.5    # otherwise truncated
                cursor[e] = 0
                ep_idx[e] += 1
        rob = rng.standard_normal((N, D)).astype(np.float32)
        steps.append((nxt, act, rew, term, done, rob))
    return init_obs, steps


def golden_replay(out):
    p = REPLAY
    buf = RecurrentOffPolicyBuffer(Box(-np.inf, np.inf, (p["obs_dim"],)), Discrete(p["n_actions"]), {}, p["n_envs"],
                                   p["buffer_size"], p["batch_size"], episode_length=p["episode_length"],
                                   lookup_length=p["lookup_length"])
    init_obs, steps = replay_stream()
    eps = [EpisodeBuffer() for _ in range(p["n_envs"])]
    for e in range(p["n_envs"]):
        eps[e].obs.append(init_obs[e])
    out["replay/init_obs"] = np.stack(init_obs)
    stored = 0
    for t, (nxt, act, rew, term, done, rob) in enumerate(steps):
        for k, v in (("next_obs", nxt), ("actions", act), ("rewards", rew), ("terminals", term), ("done", done),
                     ("reset_obs", rob)):
            out[f"replay/step{t}/{k}"] = v
        for e in range(p["n_envs"]):
            eps[e].put([nxt[e], act[e], rew[e], term[e]])
            if done[e]:
                buf.store(eps[e])
                stored += 1
                eps[e] = EpisodeBuffer()
                eps[e].obs.append(rob[e])
    assert stored > buf.n_size, stored
    out["replay/n_steps"] = np.int64(len(steps))
    out["replay/lengths"] = np.array([len(ep) for ep in buf.memory], np.int64)
    for sd in SAMPLE_SEEDS:
        np.random.seed(sd)
        s = buf.sample()
        for k in ("obs", "actions", "rewards", "terminals"):
            out[f"replay/sample{sd}/{k}"] = np.asarray(s[k])


def golden_acting(out):
    name, rnn, H, obs_dim, rep_hidden, A, seed = "act", "LSTM", 17, 5, 24, 3, 21
    N = 4
    model = build_model(rnn, H, obs_dim, rep_hidden, A, seed)
    model.load_state_dict(seeded_state(model.state_dict(), seed), strict=True)
    stand_in = SimpleNamespace(model=model, action_space=Discrete(A), n_envs=N)
    rng = np.random.default_rng(seed)
    np.random.seed(seed)
    states = model.init_rnn_states(N)
    for t in range(ACT_STEPS):
        obs = rng.standard_normal((N, obs_dim)).astype(np.float32)
        eg = (0.0, 0.5, 1.0)[t % 3]
        pol = DRQN_Agent.get_actions(stand_in, obs, eg, states)
        states = pol.auxiliary["rnn_states_next"]
        out[f"{name}/step{t}/obs"] = obs
        out[f"{name}/step{t}/egreedy"] = np.float64(eg)
        out[f"{name}/step{t}/actions"] = np.asarray(pol.env_actions, np.int64)
        out[f"{name}/step{t}/h"] = states.hidden_states.numpy().copy()
        out[f"{name}/step{t}/c"] = states.cell_states.numpy().copy()


def main():
    torch.set_num_threads(1)
    out = {}
    golden_learner(out)
    golden_replay(out)
    golden_acting(out)
    path = os.path.join(HERE, "drqn_update.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()

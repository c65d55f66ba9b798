"""Multi-agent raw environment + wrapper for the QMIX path (no SMAC / PettingZoo in this image).

``SyntheticSMACEnv`` is SMAC-SHAPED, not SMAC: the default ``5m_vs_6m`` layout is 5 agents x 72-d observations, a 98-d
global state, 12 discrete actions with an availability mask and episodes of at most 60 steps (BASELINE config 5).  The
dynamics are a cooperative cue-following task that value factorisation can actually learn, so that an agent trained
through ``REGISTRY_Agents["QMIX"]`` shows a rising score: every step each living agent is shown a cue (one-hot in the
first ``n_actions`` observation entries) naming one AVAILABLE action; the team reward is the fraction of living agents
that played their cue.  Action 0 is the SMAC "no-op": the only action of a dead agent and unavailable to a living one;
a random subset of the other actions is masked out each step; agents die at random (``agent_mask`` turns 0) and the
episode terminates when all are dead or is truncated at ``max_episode_steps``.

``XuanCeMultiAgentEnvWrapper`` mirrors xuance/environment/utils/wrapper.py:141-226: per-agent ``episode_score``,
``episode_step``, and ``agent_mask / avail_actions / state`` copied into every ``info``."""
import numpy as np

from ..common.spaces import Box, Discrete

SMAC_SHAPES = {"5m_vs_6m": dict(n_agents=5, obs_dim=72, state_dim=98, n_actions=12, episode_limit=60),
               "3m": dict(n_agents=3, obs_dim=30, state_dim=48, n_actions=9, episode_limit=60)}


class SyntheticSMACEnv:
    def __init__(self, seed=None, map_name="5m_vs_6m", n_agents=None, obs_dim=None, state_dim=None, n_actions=None,
                 episode_limit=None, p_death=0.01, p_mask=0.3):
        shp = dict(SMAC_SHAPES.get(map_name, SMAC_SHAPES["5m_vs_6m"]))
        for k, v in dict(n_agents=n_agents, obs_dim=obs_dim, state_dim=state_dim, n_actions=n_actions,
                         episode_limit=episode_limit).items():
            if v is not None:
                shp[k] = v
        self.num_agents, self.obs_dim, self.state_dim = shp["n_agents"], shp["obs_dim"], shp["state_dim"]
        self.n_actions, self.max_episode_steps = shp["n_actions"], shp["episode_limit"]
        assert self.obs_dim >= self.n_actions + 1 and self.n_actions >= 3
        self.agents = ["agent_%d" % i for i in range(self.num_agents)]
        self.agent_groups = [list(self.agents)]
        self.observation_space = {a: Box(-1.0, 1.0, (self.obs_dim,), np.float32) for a in self.agents}
        self.action_space = {a: Discrete(self.n_actions) for a in self.agents}
        self.state_space = Box(-1.0, 1.0, (self.state_dim,), np.float32)
        self.p_death, self.p_mask = p_death, p_mask
        self.rng = np.random.default_rng(seed)
        self._steps = 0
        self._alive = np.ones(self.num_agents, bool)
        self._cue = np.ones(self.num_agents, np.int64)
        self._avail = np.ones((self.num_agents, self.n_actions), bool)
        self._noise = np.zeros((self.num_agents, self.obs_dim), np.float32)

    # ---- the interface XuanCeMultiAgentEnvWrapper reads
    def get_env_info(self):
        return {"state_space": self.state_space, "observation_space": self.observation_space,
                "action_space": self.action_space, "agents": self.agents, "num_agents": self.num_agents,
                "max_episode_steps": self.max_episode_steps}

    def get_groups_info(self):
        return {"num_groups": 1, "agent_groups": self.agent_groups,
                "observation_space_groups": [self.observation_space], "action_space_groups": [self.action_space],
                "num_agents_groups": [self.num_agents]}

    def state(self):
        s = np.zeros(self.state_dim, np.float32)
        n, A = self.num_agents, self.n_actions
        s[:n] = self._alive
        k = min(self.state_dim - n, n * A)
        onehot = np.zeros((n, A), np.float32)
        onehot[np.arange(n), self._cue] = self._alive
        s[n:n + k] = onehot.reshape(-1)[:k]
        return s

    def agent_mask(self):
        return {a: bool(self._alive[i]) for i, a in enumerate(self.agents)}

    def avail_actions(self):
        return {a: self._avail[i].astype(np.int64) for i, a in enumerate(self.agents)}

    # ---- dynamics
    def _draw(self):
        n, A = self.num_agents, self.n_actions
        self._cue = self.rng.integers(1, A, size=n)
        av = self.rng.random((n, A)) >= self.p_mask
        av[:, 0] = False
        av[np.arange(n), self._cue] = True
        dead = ~self._alive
        av[dead] = False
        av[dead, 0] = True                      # a dead agent can only no-op
        self._avail = av
        self._cue[dead] = 0
        self._noise = self.rng.uniform(-0.1, 0.1, size=(n, self.obs_dim)).astype(np.float32)

    def _obs(self):
        out = {}
        for i, a in enumerate(self.agents):
            o = self._noise[i].copy()
            o[:self.n_actions] = 0.0
            if self._alive[i]:
                o[self._cue[i]] = 1.0
            o[self.n_actions] = float(self._alive[i])
            out[a] = o
        return out

    def reset(self, **kwargs):
        self._steps = 0
        self._alive[:] = True
        self._draw()
        return self._obs(), {}

    def step(self, actions):
        acts = np.array([int(actions[a]) for a in self.agents])
        alive = self._alive.copy()
        hit = (acts == self._cue) & alive
        reward = float(hit.sum()) / max(1, int(alive.sum()))
        self._steps += 1
        self._alive &= self.rng.random(self.num_agents) >= self.p_death
        terminated = not self._alive.any()
        truncated = (self._steps >= self.max_episode_steps) and not terminated
        self._draw()
        rew = {a: reward for a in self.agents}
        term = {a: bool(terminated) for a in self.agents}
        return self._obs(), rew, term, bool(truncated), {}

    def render(self, *a, **k):
        return None

    def close(self):
        pass


class XuanCeMultiAgentEnvWrapper:
    """wrapper.py:141-226."""

    def __init__(self, env, **kwargs):
        self.env = env
        self.agents, self.num_agents, self.agent_groups = env.agents, env.num_agents, env.agent_groups
        self.env_info, self.groups_info = env.get_env_info(), env.get_groups_info()
        self._episode_step = 0
        self._episode_score = {a: 0.0 for a in self.agents}

    observation_space = property(lambda self: self.env.observation_space)
    action_space = property(lambda self: self.env.action_space)
    state_space = property(lambda self: self.env.state_space)
    max_episode_steps = property(lambda self: self.env.max_episode_steps)
    state = property(lambda self: self.env.state())
    agent_mask = property(lambda self: self.env.agent_mask())
    avail_actions = property(lambda self: self.env.avail_actions())

    def _annotate(self, info):
        info["episode_step"] = self._episode_step
        info["episode_score"] = self._episode_score
        info["agent_mask"] = self.agent_mask
        info["avail_actions"] = self.avail_actions
        info["state"] = self.state
        return info

    def reset(self, **kwargs):
        obs, info = self.env.reset(**kwargs)
        self._episode_step = 0
        self._episode_score = {a: 0.0 for a in self.agents}
        return obs, self._annotate(info)

    def step(self, action):
        obs, reward, terminated, truncated, info = self.env.step(action)
        self._episode_step += 1
        for a in self.agents:
            self._episode_score[a] += reward[a]
        return obs, reward, terminated, truncated, self._annotate(info)

    def render(self, *a, **k):
        return self.env.render(*a, **k)

    def close(self):
        return self.env.close()

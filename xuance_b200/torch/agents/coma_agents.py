"""COMA agents - mirror of xuance/torch/agents/multi_agent_rl/coma_agents.py:21-650 on OnPolicyMARLAgents (the device
episode buffer and its GAE, whole-episode training with ``use_rnn``).

Acting (``get_actions``): the actor on K13, K4C ``xb_coma_act`` (epsilon-mixed sampling, epsilon on the device), the
TARGET critics on K4C critic-input rows at T = 1 with the actions just drawn, the Q of the taken actions gathered, and ONE
device-to-host read of actions, log-probabilities and values.  ``values_next`` bootstraps with the target critics and the
env's last actions (coma_agents.py:276-341); ``train_epochs`` decays epsilon (coma_agents.py:633-634) and passes it to
``COMA_Learner.update``.

Scope: one parameter-sharing group, Discrete actions (A <= 64, n <= 32), ``use_rnn=True`` with the LayerNorm Basic_RNN
whose GRU runs on K13 (one GRU layer, H <= 64, no dropout)."""
import numpy as np
import torch
import torch.nn as nn

from ... import _lib
from ..rl_models import (CategoricalActor, CounterfactualCentralizedCritic, CounterfactualMultiAgentActorCritic)
from .mappo_agents import OnPolicyMARLAgents, MARLActionOutput, MAPPO_Agents

COMA_MAX_ACTIONS, COMA_MAX_AGENTS, GRU_MAX_HIDDEN = 64, 32, 64    # K4C, K13


class COMA_Agents(OnPolicyMARLAgents):
    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        super().__init__(config, envs, num_agents, agent_keys, state_space, observation_space, action_space, callback)
        self._check_scope()
        self.start_greedy, self.end_greedy = config.start_greedy, config.end_greedy
        self.egreedy = self.start_greedy
        self.delta_egreedy = (self.start_greedy - self.end_greedy) / config.decay_step_greedy
        self.use_global_state = True
        self._eps = torch.full((1,), float(self.egreedy), dtype=torch.float32, device=self.device)
        self._eps_host = float(self.egreedy)
        self._last_actions = None
        self.model = self._build_model()
        self.memory = self._build_memory()
        self.learner = self._build_learner(self.config, self.agent_grouping, self.model, self.callback)

    def _check_scope(self):
        c = self.config
        if not all(hasattr(self.action_space[k], "n") for k in self.agent_keys):
            raise ValueError("COMA takes Discrete action spaces (Box actions have no counterfactual baseline here)")
        if len(self.group_keys) != 1:
            raise NotImplementedError("COMA: one parameter-sharing group")
        if not self.use_rnn:
            raise NotImplementedError("COMA: use_rnn=False is not supported (recurrent episodes only)")
        if getattr(c, "rnn", "GRU") != "GRU":
            raise NotImplementedError("COMA: LSTM representations are not supported (GRU only)")
        if getattr(c, "N_recurrent_layers", 1) != 1:
            raise NotImplementedError("COMA: N_recurrent_layers > 1 is not supported (one GRU layer)")
        if getattr(c, "dropout", 0) > 0:
            raise NotImplementedError("COMA: dropout > 0 is not supported")
        if c.recurrent_hidden_size > GRU_MAX_HIDDEN:
            raise NotImplementedError("COMA: recurrent_hidden_size > %d is not supported (K13), got %d"
                                      % (GRU_MAX_HIDDEN, c.recurrent_hidden_size))
        A = max(self.action_space[k].n for k in self.agent_keys)
        if A > COMA_MAX_ACTIONS:
            raise NotImplementedError("COMA: more than %d actions is not supported (K4C), got %d" % (COMA_MAX_ACTIONS, A))
        if self.n_agents > COMA_MAX_AGENTS:
            raise NotImplementedError("COMA: more than %d agents is not supported (K4C), got %d"
                                      % (COMA_MAX_AGENTS, self.n_agents))

    _build_agent_feature_encoder = MAPPO_Agents._build_agent_feature_encoder

    def _build_model(self):
        """coma_agents.py:49-115."""
        actors, critic_encoders = nn.ModuleDict(), nn.ModuleDict()
        for group_key, group_agents in self.groups.items():
            ref = group_agents[0]
            enc = lambda: self._build_agent_feature_encoder(self.config.representation, group_agents,
                                                            self.observation_space[ref])
            actors[group_key] = CategoricalActor(representation=enc(), actor_hidden_size=self.config.actor_hidden_size,
                                                 action_space=self.action_space[ref], normalizer=self.normalize_fn,
                                                 initializer=self.initializer, activation=self.activation,
                                                 device=self.device)
            critic_encoders[group_key] = enc()
        critic = CounterfactualCentralizedCritic(
            grouping=self.agent_grouping, representations=critic_encoders, state_space=self.state_space,
            action_space=self.action_space, critic_hidden_size=self.config.critic_hidden_size,
            normalizer=self.normalize_fn, initializer=self.initializer, activation=self.activation,
            use_rnn=self.use_rnn, device=self.device)
        return CounterfactualMultiAgentActorCritic(grouping=self.agent_grouping, actors=actors, critics=critic,
                                                  use_rnn=self.use_rnn, device=self.device).to(self.device)

    def store_experience(self, obs_list, avail_actions, actions_list, log_pi_a, rewards_list, values_dict,
                         terminals_list, info, **kwargs):
        """coma_agents.py:117-173: every agent stores the agent-mean team reward."""
        team = [np.array(list(d.values())).mean() for d in rewards_list]
        rewards = [{k: team[e] for k in self.agent_keys} for e in range(len(rewards_list))]
        super().store_experience(obs_list, avail_actions, actions_list, log_pi_a, rewards, values_dict, terminals_list,
                                 info, **kwargs)

    def _state_rows(self, state, n_envs):
        return torch.as_tensor(np.asarray(state, np.float32), device=self.device).reshape(n_envs, -1)

    @torch.no_grad()
    def get_actions(self, obs_list, state=None, avail_actions_list=None, rnn_states_actor=None,
                    rnn_states_critic=None, test_mode=False, deterministic=False, **kwargs):
        """coma_agents.py:175-273."""
        n_envs, K = len(obs_list), self.agent_keys
        obs, avail = self._build_inputs(obs_list, avail_actions_list)
        obs_d = torch.from_numpy(obs).to(self.device)
        if self.use_rnn:
            logits, rnn_states_actor = self.model.logits(obs_d, rnn_states=rnn_states_actor, return_states=True)
        else:
            logits = self.model.logits(obs_d)
        logits = logits.contiguous()
        R, A = logits.shape
        av = None if avail is None else torch.from_numpy(avail).to(self.device)
        out = torch.empty((3, R), dtype=torch.float32, device=self.device)   # actions, log_pi, values
        acts_i = torch.empty(R, dtype=torch.int32, device=self.device)
        u = None if deterministic else torch.rand(R, device=self.device)
        if not test_mode and self._eps_host != float(self.egreedy):
            self._eps.fill_(float(self.egreedy))
            self._eps_host = float(self.egreedy)
        _lib.call("xb_coma_act", _lib.ptr(logits), _lib.ptr(av), 0 if av is None else av.shape[1],
                  None if test_mode else _lib.ptr(self._eps), _lib.ptr(u), R, A, _lib.ptr(out[0]), _lib.ptr(acts_i),
                  _lib.ptr(out[1]))
        if not test_mode:           # the target critics' Q of the taken actions (coma_agents.py:237-261)
            q, rnn_states_critic = self.model.q_values(self._state_rows(state, n_envs), obs_d,
                                                       out[0].reshape(n_envs, len(K)), rnn_states_critic,
                                                       return_states=True, target=True)
            out[2] = q.gather(1, acts_i.long().unsqueeze(1)).squeeze(1)
        host = out.cpu().numpy().reshape(3, n_envs, len(K))
        actions_list = [{k: int(host[0, e, i]) for i, k in enumerate(K)} for e in range(n_envs)]
        self._last_actions = actions_list
        log_pi, values = {}, {}
        if not test_mode:
            log_pi = {k: host[1, :, i].copy() for i, k in enumerate(K)}
            values = {k: host[2, :, i].copy() for i, k in enumerate(K)}
        return MARLActionOutput(env_actions=actions_list, log_probs=log_pi, values=values,
                                rnn_states_actor=rnn_states_actor, rnn_states_critic=rnn_states_critic)

    @torch.no_grad()
    def values_next(self, i_env, obs_dict, state=None, actions_n=None, rnn_states_critic=None):
        """coma_agents.py:275-341: the target critics' Q of env i_env's last actions (``actions_n``; by default the
        actions get_actions last chose for that env) at its next observation and state."""
        K = self.agent_keys
        acts = self._last_actions[i_env] if actions_n is None else actions_n
        obs, _ = self._build_inputs([obs_dict])
        h = None
        if self.use_rnn:
            n = len(K)
            h = rnn_states_critic[:, i_env * n:(i_env + 1) * n]
        a = torch.tensor([[float(acts[k]) for k in K]], dtype=torch.float32, device=self.device)
        q = self.model.q_values(self._state_rows(state, 1), torch.from_numpy(obs).to(self.device), a, h, target=True)
        v = q.gather(1, a.reshape(-1, 1).long()).reshape(-1).cpu().numpy()
        return None, {k: v[i] for i, k in enumerate(K)}

    def train_epochs(self, n_epochs=1):
        """coma_agents.py:618-650: epsilon decays with the step count (until it first falls below end_greedy), then
        the shuffled minibatch updates with that epsilon."""
        if self.egreedy >= self.end_greedy:
            self.egreedy = self.start_greedy - self.delta_egreedy * self.current_step
        info_train = {}
        if self.memory.full:
            indexes = np.arange(self.buffer_size)
            for e in range(n_epochs):
                np.random.shuffle(indexes)
                for start in range(0, self.buffer_size, self.batch_size):
                    last = e == n_epochs - 1 and start + self.batch_size >= self.buffer_size
                    info_train = self.learner.update(self.memory.sample(indexes[start:start + self.batch_size]),
                                                     self.egreedy, sync=last)
            self.callback.on_train_epochs_end(self.current_step, policy=self.model, memory=self.memory,
                                              current_episode=self.current_episode, n_epochs=n_epochs,
                                              buffer_size=self.buffer_size, update_info=info_train)
            self.memory.clear()
        info_train["epsilon-greedy"] = self.egreedy
        return info_train

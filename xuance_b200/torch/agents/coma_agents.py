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
from ..rl_models.gru import check_scope
from .mappo_agents import OnPolicyMARLAgents

COMA_MAX_ACTIONS, COMA_MAX_AGENTS = 64, 32    # K4C


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
        if not all(hasattr(self.action_space[k], "n") for k in self.agent_keys):
            raise ValueError("COMA takes Discrete action spaces (Box actions have no counterfactual baseline here)")
        if len(self.group_keys) != 1:
            raise NotImplementedError("COMA: one parameter-sharing group")
        if not self.use_rnn:
            raise NotImplementedError("COMA: use_rnn=False is not supported (recurrent episodes only)")
        check_scope("COMA", self.config)
        A = max(self.action_space[k].n for k in self.agent_keys)
        if A > COMA_MAX_ACTIONS:
            raise NotImplementedError("COMA: more than %d actions is not supported (K4C), got %d" % (COMA_MAX_ACTIONS, A))
        if self.n_agents > COMA_MAX_AGENTS:
            raise NotImplementedError("COMA: more than %d agents is not supported (K4C), got %d"
                                      % (COMA_MAX_AGENTS, self.n_agents))

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

    def get_actions(self, *args, **kwargs):
        """coma_agents.py:175-273; remembers the actions for ``values_next``."""
        policy_out = super().get_actions(*args, **kwargs)
        self._last_actions = policy_out.env_actions
        return policy_out

    def _act(self, obs_d, logits, avail, state, n_envs, rnn_states_critic, test_mode, deterministic):
        """K4C's epsilon-mixed sampling, then the target critics' Q of the taken actions."""
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
                                                       out[0].reshape(n_envs, self.n_agents), rnn_states_critic,
                                                       return_states=True, target=True)
            out[2] = q.gather(1, acts_i.long().unsqueeze(1)).squeeze(1)
        return out, rnn_states_critic

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
        info_train = super().train_epochs(n_epochs)
        info_train["epsilon-greedy"] = self.egreedy
        return info_train

    def _update(self, sample, sync):
        return self.learner.update(sample, self.egreedy, sync=sync)

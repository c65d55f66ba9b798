"""VDAC and IAC agents - mirrors of xuance/torch/agents/multi_agent_rl/vdac_agents.py:308-560 and iac_agents.py:578-772 on
OnPolicyMARLAgents (acting through K10, the device episode buffer and its GAE, whole-episode training with ``use_rnn``).

Scope: one parameter-sharing group, Discrete actions, Basic_MLP representations or, with ``use_rnn=True``, the LayerNorm
Basic_RNN whose GRU runs on K13 (one GRU layer, H <= 64).  VDAC mixes with VDN (the sum, inside K4V) or QMIX (K9 mix,
n <= 16 agents)."""
import numpy as np
import torch
import torch.nn as nn

from ..rl_models import (CategoricalActor, StateValueCritic, QMIX_Mixer, VDN_mixer, IndependentActorCritic,
                         ValueDecompositionActorCritic)
from .mappo_agents import OnPolicyMARLAgents

QMIX_MAX_AGENTS = 16     # K9 mix (xb_qmix_mix_fwd / _bwd)


class IAC_Agents(OnPolicyMARLAgents):
    """iac_agents.py:578-772: independent actors and critics; the value of each agent is its own V_i."""

    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        super().__init__(config, envs, num_agents, agent_keys, state_space, observation_space, action_space, callback)
        if not all(hasattr(self.action_space[k], "n") for k in self.agent_keys):
            raise NotImplementedError("%s takes Discrete action spaces (Box actions are not supported)"
                                      % type(self).__name__)
        self._check_scope()
        self.model = self._build_model()
        self.memory = self._build_memory()
        self.learner = self._build_learner(self.config, self.agent_grouping, self.model, self.callback)

    def _check_scope(self):
        pass

    def _actors_critics(self):
        actors, critics = nn.ModuleDict(), nn.ModuleDict()
        for group_key, group_agents in self.groups.items():
            ref = group_agents[0]
            enc = lambda: self._build_agent_feature_encoder(self.config.representation, group_agents,
                                                            self.observation_space[ref])
            actors[group_key] = CategoricalActor(representation=enc(), actor_hidden_size=self.config.actor_hidden_size,
                                                 action_space=self.action_space[ref], normalizer=self.normalize_fn,
                                                 initializer=self.initializer, activation=self.activation,
                                                 device=self.device)
            critics[group_key] = StateValueCritic(representation=enc(),
                                                  critic_hidden_size=self.config.critic_hidden_size,
                                                  normalizer=self.normalize_fn, initializer=self.initializer,
                                                  activation=self.activation, device=self.device)
        return actors, critics

    def _build_model(self):
        actors, critics = self._actors_critics()
        return IndependentActorCritic(grouping=self.agent_grouping, actors=actors, critics=critics,
                                      use_rnn=self.use_rnn, device=self.device).to(self.device)

    def store_experience(self, obs_list, avail_actions, actions_list, log_pi_a, rewards_list, values_dict,
                         terminals_list, info, **kwargs):
        """vdac_agents.py:415-448 / iac_agents.py:671-704: every agent stores the agent-mean team reward, and no
        log_pi_old (the buffer's field holds zeros, which nothing reads)."""
        team = [np.array(list(d.values())).mean() for d in rewards_list]
        rewards = [{k: team[e] for k in self.agent_keys} for e in range(len(rewards_list))]
        zeros = {k: np.zeros(len(rewards_list), np.float32) for k in self.agent_keys}
        super().store_experience(obs_list, avail_actions, actions_list, zeros, rewards, values_dict, terminals_list,
                                 info, **kwargs)


class VDAC_Agents(IAC_Agents):
    """vdac_agents.py:308-560: the critics' V_i mixed into V_tot, which acting and bootstrapping broadcast to every
    agent."""

    def _check_scope(self):
        self.mixer = getattr(self.config, "mixer", "VDN")
        if self.mixer not in ("VDN", "QMIX"):
            raise NotImplementedError("VDAC: mixer %r is not supported (VDN or QMIX)" % (self.mixer,))
        if self.mixer == "QMIX":
            if self.n_agents > QMIX_MAX_AGENTS:
                raise NotImplementedError("VDAC with mixer: QMIX supports up to %d agents (K9 mix), got %d"
                                          % (QMIX_MAX_AGENTS, self.n_agents))
            self.use_global_state = True        # vdac_agents.py:398

    def _build_model(self):
        actors, critics = self._actors_critics()
        if self.mixer == "VDN":
            mixer = VDN_mixer()
        else:
            mixer = QMIX_Mixer(self.state_space.shape[-1], self.config.hidden_dim_mixing_net,
                               self.config.hidden_dim_hyper_net, self.n_agents, self.device)
        return ValueDecompositionActorCritic(grouping=self.agent_grouping, actors=actors, critics=critics, mixer=mixer,
                                             use_rnn=self.use_rnn, device=self.device).to(self.device)

    def _critic_values(self, obs_d, state, n_envs, rnn_states=None, return_states=False):
        """V_tot of each env, repeated for its agents (vdac_agents.py:503-512, 540-558)."""
        n = self.n_agents
        v, h = self.model.values(obs_d, rnn_states=rnn_states, return_states=True)
        st = None
        if self.use_global_state and state is not None:
            st = torch.as_tensor(np.asarray(state, np.float32), device=self.device).reshape(n_envs, -1)
        v = self.model.values_tot(v.reshape(n_envs, n), st).reshape(n_envs).repeat_interleave(n)
        return (v, h) if return_states else v

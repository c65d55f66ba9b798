"""IQL agents - mirror of xuance/torch/agents/multi_agent_rl/iql_agents.py:12-84 on OffPolicyMARLAgents (the episode
replay, epsilon-greedy acting, whole-episode training with ``use_rnn``).

The model is a MixingQNetwork of DiscreteActionValueCritic agents over Basic_RNN_K13 (the GRU runs on K13) with the
parameter-free IndependentMixer, so a reference state_dict loads with strict=True.  The epsilon schedule is IQL's own,
(start_greedy - end_greedy) / decay_step_greedy per environment step (iql_agents.py:37), not QMIX's per-vector-step one.

Scope: one parameter-sharing group, Discrete actions (A <= 64, n <= 32, K9I), ``use_rnn=True`` with one GRU layer of
H <= 64 (K13)."""
import torch.nn as nn

from ..rl_models import (ActivationFunctions, AgentFeatureEncoder, Basic_RNN_K13, DiscreteActionValueCritic,
                         IndependentMixer, MixingQNetwork)
from ...common import space2shape
from .marl import OffPolicyMARLAgents

IQL_MAX_ACTIONS, IQL_MAX_AGENTS, GRU_MAX_HIDDEN = 64, 32, 64    # K9I, K13


class IQL_Agents(OffPolicyMARLAgents):
    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        super().__init__(config, envs, num_agents, agent_keys, state_space, observation_space, action_space, callback)
        self._check_scope()
        self.start_greedy, self.end_greedy = config.start_greedy, config.end_greedy
        self.delta_egreedy = (self.start_greedy - self.end_greedy) / config.decay_step_greedy
        self.e_greedy = self.start_greedy
        self.model = self._build_model()
        self.memory = self._build_memory()
        self.learner = self._build_learner(self.config, self.agent_grouping, self.model, self.callback)

    def _check_scope(self):
        c = self.config
        if not all(hasattr(self.action_space[k], "n") for k in self.agent_keys):
            raise ValueError("IQL takes Discrete action spaces (Box actions have no Q-value head here)")
        if len(self.group_keys) != 1:
            raise NotImplementedError("IQL: one parameter-sharing group")
        if not self.use_rnn:
            raise NotImplementedError("IQL: use_rnn=False is not supported (recurrent episodes only)")
        if getattr(c, "rnn", "GRU") != "GRU":
            raise NotImplementedError("IQL: LSTM representations are not supported (GRU only)")
        if getattr(c, "N_recurrent_layers", 1) != 1:
            raise NotImplementedError("IQL: N_recurrent_layers > 1 is not supported (one GRU layer)")
        if getattr(c, "dropout", 0) > 0:
            raise NotImplementedError("IQL: dropout > 0 is not supported")
        if c.recurrent_hidden_size > GRU_MAX_HIDDEN:
            raise NotImplementedError("IQL: recurrent_hidden_size > %d is not supported (K13), got %d"
                                      % (GRU_MAX_HIDDEN, c.recurrent_hidden_size))
        A = max(self.action_space[k].n for k in self.agent_keys)
        if A > IQL_MAX_ACTIONS:
            raise NotImplementedError("IQL: more than %d actions is not supported (K9I), got %d" % (IQL_MAX_ACTIONS, A))
        if self.n_agents > IQL_MAX_AGENTS:
            raise NotImplementedError("IQL: more than %d agents is not supported (K9I), got %d"
                                      % (IQL_MAX_AGENTS, self.n_agents))
        if getattr(c, "qmix_rnn_detach_q_eval", False):
            raise NotImplementedError("IQL: qmix_rnn_detach_q_eval=True would detach the only trained term (there is "
                                      "no mixer), so nothing would train")

    def _build_q_networks(self):
        cfg = self.config
        q_networks = nn.ModuleDict()
        for group_key, group_agents in self.groups.items():
            ref = group_agents[0]
            rep = Basic_RNN_K13(input_shape=space2shape(self.observation_space[ref]),
                                hidden_sizes=getattr(cfg, "representation_hidden_size", None), normalize=None,
                                initialize=nn.init.orthogonal_, activation=ActivationFunctions[cfg.activation],
                                fc_hidden_sizes=cfg.fc_hidden_sizes, N_recurrent_layers=cfg.N_recurrent_layers,
                                recurrent_hidden_size=cfg.recurrent_hidden_size, rnn=cfg.rnn, dropout=cfg.dropout,
                                device=self.device)
            q_networks[group_key] = DiscreteActionValueCritic(
                representation=AgentFeatureEncoder(rep), action_space=self.action_space[ref],
                critic_hidden_size=cfg.q_hidden_size, normalizer=self.normalize_fn, initializer=self.initializer,
                activation=self.activation, device=self.device)
        return q_networks

    def _build_model(self):
        """iql_agents.py:44-84."""
        return MixingQNetwork(grouping=self.agent_grouping, q_networks=self._build_q_networks(),
                              mixer=IndependentMixer(), use_rnn=self.use_rnn, device=self.device).to(self.device)

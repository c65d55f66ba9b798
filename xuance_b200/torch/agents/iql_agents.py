"""IQL agents - mirror of xuance/torch/agents/multi_agent_rl/iql_agents.py:12-84 on OffPolicyMARLAgents (the episode
replay, epsilon-greedy acting, whole-episode training with ``use_rnn``).

The model is a MixingQNetwork of DiscreteActionValueCritic agents over Basic_RNN_K13 (the GRU runs on K13) with the
parameter-free IndependentMixer, so a reference state_dict loads with strict=True.  The epsilon schedule is IQL's own,
(start_greedy - end_greedy) / decay_step_greedy per environment step (iql_agents.py:37), not QMIX's per-vector-step one.

Scope: one parameter-sharing group, Discrete actions (A <= 64, n <= 32, K9I), ``use_rnn=True`` with one GRU layer of
H <= 64 (K13)."""
from ..rl_models import IndependentMixer, MixingQNetwork
from ..rl_models.gru import check_scope
from .marl import OffPolicyMARLAgents

IQL_MAX_ACTIONS, IQL_MAX_AGENTS = 64, 32    # K9I


class IQL_Agents(OffPolicyMARLAgents):
    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        super().__init__(config, envs, num_agents, agent_keys, state_space, observation_space, action_space, callback)
        self._check_scope()
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
        check_scope("IQL", c)
        A = max(self.action_space[k].n for k in self.agent_keys)
        if A > IQL_MAX_ACTIONS:
            raise NotImplementedError("IQL: more than %d actions is not supported (K9I), got %d" % (IQL_MAX_ACTIONS, A))
        if self.n_agents > IQL_MAX_AGENTS:
            raise NotImplementedError("IQL: more than %d agents is not supported (K9I), got %d"
                                      % (IQL_MAX_AGENTS, self.n_agents))
        if getattr(c, "qmix_rnn_detach_q_eval", False):
            raise NotImplementedError("IQL: qmix_rnn_detach_q_eval=True would detach the only trained term (there is "
                                      "no mixer), so nothing would train")

    def _build_agent_feature_encoder(self, representation_choice, group_agents, input_space):
        return self._build_k13_encoder(input_space, None)

    def _build_model(self):
        """iql_agents.py:44-84."""
        return MixingQNetwork(grouping=self.agent_grouping, q_networks=self._build_q_networks(),
                              mixer=IndependentMixer(), use_rnn=self.use_rnn, device=self.device).to(self.device)

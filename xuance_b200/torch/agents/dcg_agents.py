"""DCG agents - mirror of xuance/torch/agents/multi_agent_rl/dcg_agents.py:16-155."""
import torch.nn as nn

from ..rl_models import ValueHead, DCG_Utility, DCG_Payoff, Coordination_Graph, DeepCoordinationGraph
from ..rl_models.dcg import check_graph_limits
from .marl import OffPolicyMARLAgents


class DCG_Agents(OffPolicyMARLAgents):
    """dcg_agents.py:16-155 (DCG and DCG_S): the off-policy MARL rollout loop and episode replay with a
    DeepCoordinationGraph whose agents are K13 GRUs.  Acting is one GRU step, both heads and the K9C greedy on the
    device, then one copy of the actions to the host.

    Exploration: the reference sets delta_egreedy = (start - end) / decay_step_greedy but never initialises e_greedy, so
    it never explores.  This runs the evidently intended computation: e_greedy starts at start_greedy and decays by that
    delta per environment step (DESIGN.md "Reference quirks")."""

    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        if not getattr(config, "use_rnn", False):
            raise NotImplementedError("hot-path scope: DCG with use_rnn=True (the sc2 configurations)")
        if getattr(config, "rnn", "GRU") != "GRU":
            raise NotImplementedError("DCG: LSTM representations are not supported (GRU only)")
        super().__init__(config, envs, num_agents, agent_keys, state_space, observation_space, action_space, callback)
        self.use_global_state = config.agent == "DCG_S"
        if self.use_global_state and self.state_space is None:
            raise ValueError("DCG_S evaluates V(s) on the global state: provide envs or state_space")
        self.model = self._build_model()
        self.memory = self._build_memory()
        self.learner = self._build_learner(self.config, self.agent_grouping, self.model, self.callback)

    def _build_model(self):
        cfg = self.config
        n_act = max(self.action_space[k].n for k in self.agent_keys)
        graph = Coordination_Graph(self.n_agents, cfg.graph_type, self.device)
        check_graph_limits(self.n_agents, n_act, graph.n_edges)
        graph.set_coordination_graph()
        representations = nn.ModuleDict()
        for group_key, group_agents in self.groups.items():
            representations[group_key] = self._build_k13_encoder(self.observation_space[group_agents[0]], None)
        H = cfg.recurrent_hidden_size
        utility = DCG_Utility(H, cfg.hidden_utility_dim, n_act, self.device)
        payoffs = DCG_Payoff(2 * H, cfg.hidden_payoff_dim, n_act, cfg.low_rank_payoff, cfg.payoff_rank, self.device)
        bias = None
        if self.use_global_state:
            bias = ValueHead(feature_dim=self.state_space.shape[0], hidden_size=cfg.hidden_bias_dim,
                             normalizer=self.normalize_fn, initializer=self.initializer, activation=self.activation,
                             device=self.device)
        return DeepCoordinationGraph(grouping=self.agent_grouping, action_space=self.action_space,
                                     representation=representations, utility=utility, payoffs=payoffs,
                                     dcg_graph=graph, dcg_s=self.use_global_state, bias=bias, use_rnn=self.use_rnn,
                                     device=self.device, n_msg_iterations=cfg.n_msg_iterations,
                                     msg_normalized=cfg.msg_normalized).to(self.device)

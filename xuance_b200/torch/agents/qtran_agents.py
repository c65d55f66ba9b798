"""QTRAN agents - mirror of xuance/torch/agents/multi_agent_rl/qtran_agents.py:17-101."""
from ..rl_models import VDN_mixer, QTRAN_Base, QTRAN_Alt, QTranMixingNetwork
from ..rl_models.qtran import check_limits
from .marl import QMIX_Agents


class QTRAN_Agents(QMIX_Agents):
    """qtran_agents.py:17-101 (QTRAN_base and QTRAN_alt): QMIX's acting, epsilon-greedy exploration and episode replay,
    with a QTranMixingNetwork whose agents are K13 GRUs and whose joint network is QTRAN_Base or QTRAN_Alt."""

    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        if not getattr(config, "use_rnn", False):
            raise NotImplementedError("hot-path scope: QTRAN with use_rnn=True (the sc2 configurations)")
        if getattr(config, "rnn", "GRU") != "GRU":
            raise NotImplementedError("QTRAN: LSTM representations are not supported (GRU only)")
        if config.agent not in ("QTRAN_base", "QTRAN_alt"):
            raise ValueError("Mixer {} not recognised.".format(config.agent))
        # the reference sizes the encoder from q_hidden_size[0] and feeds it the GRU output (recurrent_hidden_size)
        if config.q_hidden_size[0] != config.recurrent_hidden_size:
            raise ValueError("QTRAN encodes the GRU outputs: q_hidden_size[0] (%d) must equal recurrent_hidden_size (%d)"
                             % (config.q_hidden_size[0], config.recurrent_hidden_size))
        super().__init__(config, envs, num_agents, agent_keys, state_space, observation_space, action_space, callback)

    def _build_agent_feature_encoder(self, representation_choice, group_agents, input_space):
        return self._build_k13_encoder(input_space, None)

    def _build_model(self):
        cfg = self.config
        n_act = max(self.action_space[k].n for k in self.agent_keys)
        check_limits(self.n_agents, n_act, cfg.recurrent_hidden_size)
        q_networks = self._build_q_networks()
        head = QTRAN_Base if cfg.agent == "QTRAN_base" else QTRAN_Alt
        qtran_mixer = head(dim_state=self.state_space.shape[-1], action_space=self.action_space,
                           dim_hidden=cfg.qtran_net_hidden_dim, n_agents=self.n_agents,
                           dim_utility_hidden=cfg.q_hidden_size[0], use_parameter_sharing=self.use_parameter_sharing,
                           device=self.device)
        return QTranMixingNetwork(grouping=self.agent_grouping, q_networks=q_networks, mixer=VDN_mixer(),
                                  qtran_mixer=qtran_mixer, use_rnn=self.use_rnn, device=self.device).to(self.device)

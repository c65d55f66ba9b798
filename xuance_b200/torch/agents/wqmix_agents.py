"""Weighted QMIX agents - mirror of xuance/torch/agents/multi_agent_rl/wqmix_agents.py:12-88."""
from ..rl_models import QMIX_FF_Mixer, WeightedMixingQNetwork
from .marl import QMIX_Agents


class WQMIX_Agents(QMIX_Agents):
    """wqmix_agents.py:12-88 (OW-QMIX and CW-QMIX): QMIX's acting, epsilon-greedy exploration and episode replay, with the
    WeightedMixingQNetwork (central agent networks and the feed-forward mixer of hidden_dim_ff_mix_net units)."""

    def _build_model(self):
        q_networks = self._build_q_networks()
        mixer = self._build_mixer()
        ff_mixer = QMIX_FF_Mixer(dim_state=self.state_space.shape[0], dim_hidden=self.config.hidden_dim_ff_mix_net,
                                 n_agents=self.n_agents, device=self.device)
        return WeightedMixingQNetwork(grouping=self.agent_grouping, q_networks=q_networks, mixer=mixer, ff_mixer=ff_mixer,
                                      use_rnn=self.use_rnn, device=self.device).to(self.device)

"""C51 / QR-DQN agents - mirrors of xuance/torch/agents/qlearning_family/c51_agent.py:10-47 and qrdqn_agent.py:10-45:
DQN_Agent's replay, epsilon-greedy schedule (OffPolicyAgent.exploration, torch's random stream) and training loop, with
C51DeepQNetwork / QRDeepQNetwork, whose greedy actions come from the K6Z ``xb_dist_greedy`` launch."""
import numpy as np
import torch

from ...common.spaces import is_discrete
from ..rl_models import C51DeepQNetwork, QRDeepQNetwork, ActionOutput
from .dqn_agent import DQN_Agent


class _DistDQN_Agent(DQN_Agent):
    def __init__(self, config, envs=None, observation_space=None, action_space=None, callback=None):
        if getattr(config, "use_actions_mask", False):
            raise NotImplementedError("%s does not support action masks (use_actions_mask=True)" % type(self).__name__)
        if not is_discrete(envs.action_space if envs is not None else action_space):
            raise ValueError('action_space must be Discrete')
        super().__init__(config, envs, observation_space, action_space, callback)

    @torch.no_grad()
    def get_actions(self, observations, test_mode=False):
        """OffPolicyAgent.get_actions with the greedy actions from ``greedy_actions``: acting reads only the actions, so
        C51's [B, A, N] probabilities are not written."""
        if isinstance(observations, np.ndarray):
            observations = torch.from_numpy(observations).to(self.device)
        actions = self.model.greedy_actions(observations)
        if not test_mode:
            actions = self.exploration(actions)
        return ActionOutput(env_actions=actions.detach().cpu().numpy())


class C51_Agent(_DistDQN_Agent):
    def _build_model(self):
        rep = self._build_representation(self.config.representation, self.observation_space, self.config)
        return C51DeepQNetwork(representation=rep, hidden_size=self.config.q_hidden_size, action_space=self.action_space,
                               atom_num=self.config.atom_num, v_min=self.config.v_min, v_max=self.config.v_max,
                               normalizer=self.normalize_fn, initializer=self.initializer, activation=self.activation,
                               device=self.device).to(self.device)


class QRDQN_Agent(_DistDQN_Agent):
    def _build_model(self):
        rep = self._build_representation(self.config.representation, self.observation_space, self.config)
        return QRDeepQNetwork(representation=rep, hidden_size=self.config.q_hidden_size, action_space=self.action_space,
                              quantile_num=self.config.quantile_num, normalizer=self.normalize_fn,
                              initializer=self.initializer, activation=self.activation,
                              device=self.device).to(self.device)

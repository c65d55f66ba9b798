"""SAC agent - mirror of xuance/torch/agents/policy_gradient/sac_agent.py:19-103.

A Box action space builds SAC_GaussianActor / TwinActionValueCritic / SoftActorCritic (learner "SAC_Learner"); a Discrete one
builds CategoricalActor / TwinDiscreteActionValueCritic / SoftActorCriticDiscrete (SAC-Discrete, learner "SACDIS_Learner",
policy "Categorical_SAC"), whose actions K10 samples on the device."""
from copy import deepcopy

import numpy as np
import torch

from ...common.spaces import is_discrete
from ..rl_models import (SAC_GaussianActor, TwinActionValueCritic, SoftActorCritic, CategoricalActor,
                         TwinDiscreteActionValueCritic, SoftActorCriticDiscrete, ActivationFunctions, ActionOutput)
from .off_policy import OffPolicyAgent


class SAC_Agent(OffPolicyAgent):
    def __init__(self, config, envs=None, observation_space=None, action_space=None, callback=None):
        super().__init__(config, envs, observation_space, action_space, callback)
        self.model = self._build_model()
        self.memory = self._build_memory()
        self.learner = self._build_learner(self.config, self.model, self.callback)

    def _build_model(self):
        if is_discrete(self.action_space):
            return self._build_discrete_model()
        if not hasattr(self.action_space, "low"):
            raise NotImplementedError("SAC takes Box or Discrete action spaces, not %r" % (self.action_space,))
        rep = self._build_representation(self.config.representation, self.observation_space, self.config)
        actor = SAC_GaussianActor(representation=rep, actor_hidden_size=self.config.actor_hidden_size,
                                  action_space=self.action_space, normalizer=self.normalize_fn,
                                  initializer=self.initializer, activation=self.activation,
                                  activation_action=ActivationFunctions[self.config.activation_action],
                                  device=self.device)
        critic = TwinActionValueCritic(representation=deepcopy(rep), action_space=self.action_space,
                                       critic_hidden_size=self.config.critic_hidden_size, normalizer=self.normalize_fn,
                                       initializer=self.initializer, activation=self.activation, device=self.device)
        return SoftActorCritic(actor=actor, critic=critic).to(self.device)

    def _build_discrete_model(self):
        if self.use_actions_mask:
            raise NotImplementedError("discrete SAC with action masks (use_actions_mask=True) is not supported")
        if self.config.representation == "Basic_CNN" or getattr(self.config, "env_name", None) == "Atari":
            raise NotImplementedError("discrete SAC on Atari (sac/atari.yaml: Basic_CNN with leaky_relu, image replay) "
                                      "is not supported")
        if self.action_space.n > 64:
            raise NotImplementedError("discrete SAC supports at most 64 actions (K8D), got %d" % self.action_space.n)
        rep = self._build_representation(self.config.representation, self.observation_space, self.config)
        actor = CategoricalActor(representation=rep, actor_hidden_size=self.config.actor_hidden_size,
                                 action_space=self.action_space, normalizer=self.normalize_fn,
                                 initializer=self.initializer, activation=self.activation, device=self.device)
        critic = TwinDiscreteActionValueCritic(representation=deepcopy(rep), action_space=self.action_space,
                                               critic_hidden_size=self.config.critic_hidden_size,
                                               normalizer=self.normalize_fn, initializer=self.initializer,
                                               activation=self.activation, device=self.device)
        return SoftActorCriticDiscrete(actor=actor, critic=critic).to(self.device)

    @torch.no_grad()
    def get_actions(self, observations, test_mode=False):
        """Box: the squashed Gaussian's sample, or its mean in test mode.  Discrete: a K10 sample of the categorical
        policy, or its first argmax in test mode (the reference samples in test mode too)."""
        if isinstance(observations, np.ndarray):
            observations = torch.from_numpy(observations).to(self.device)
        actions = self.model.act(observations, deterministic=test_mode)
        return ActionOutput(env_actions=actions.cpu().numpy())

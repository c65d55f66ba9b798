"""DDPG and TD3 agents - mirror of xuance/torch/agents/policy_gradient/ddpg_agent.py:13-69 and td3_agent.py:13-66.

A Box action space (one dimension of action components) builds DeterministicActor / ActionValueCritic /
DeterministicActorCritic (DDPG, learner "DDPG_Learner") or DeterministicActor / TwinActionValueCritic /
TwinDelayedActorCritic (TD3, learner "TD3_Learner").  Exploration adds scaled Gaussian noise to the actor's output and
clamps it to the environment's bounds in one K8T ``xb_perturb_actions`` launch."""
from copy import deepcopy

import numpy as np
import torch

from ... import _lib
from ...common.spaces import is_discrete
from ..rl_models import (DeterministicActor, ActionValueCritic, TwinActionValueCritic, DeterministicActorCritic,
                         TwinDelayedActorCritic, ActivationFunctions, ActionOutput)
from .off_policy import OffPolicyAgent

_NO_SIMULATOR = {"MuJoCo": "MuJoCo", "Box2D": "Box2D", "Drones": "drone (gym-pybullet-drones)"}


class DDPG_Agent(OffPolicyAgent):
    def __init__(self, config, envs=None, observation_space=None, action_space=None, callback=None):
        super().__init__(config, envs, observation_space, action_space, callback)
        if is_discrete(self.action_space) or not hasattr(self.action_space, "low"):
            raise ValueError('action_space must be Box')
        if len(self.action_space.shape) != 1:
            raise NotImplementedError("%s takes a one-dimensional Box action space, got shape %s"
                                      % (type(self).__name__, tuple(self.action_space.shape)))
        env_name = getattr(config, "env_name", None)
        if env_name in _NO_SIMULATOR:
            raise NotImplementedError("%s configs are not supported: the %s simulator is not part of this package"
                                      % (env_name, _NO_SIMULATOR[env_name]))
        if getattr(config, "device_rollout", False):
            raise NotImplementedError("a device-side off-policy rollout (device_rollout=True) is not supported")
        # ddpg_agent.py:31-33: the noise decays over running_steps / n_envs vector steps
        self.start_noise, self.end_noise = config.start_noise, config.end_noise
        self.noise_scale = config.start_noise
        self.delta_noise = (self.start_noise - self.end_noise) / (config.running_steps / self.n_envs)
        self._act_low = torch.as_tensor(self.action_space.low, dtype=torch.float32, device=self.device)
        self._act_high = torch.as_tensor(self.action_space.high, dtype=torch.float32, device=self.device)
        self.model = self._build_model()
        self.memory = self._build_memory()
        self.learner = self._build_learner(self.config, self.model, self.callback)

    def _actor(self, rep):
        return DeterministicActor(representation=rep, actor_hidden_size=self.config.actor_hidden_size,
                                  action_space=self.action_space, normalizer=self.normalize_fn,
                                  initializer=self.initializer, activation=self.activation,
                                  activation_action=ActivationFunctions[self.config.activation_action],
                                  device=self.device)

    def _build_model(self):
        rep = self._build_representation(self.config.representation, self.observation_space, self.config)
        critic = ActionValueCritic(representation=deepcopy(rep), action_space=self.action_space,
                                   critic_hidden_size=self.config.critic_hidden_size, normalizer=self.normalize_fn,
                                   initializer=self.initializer, activation=self.activation, device=self.device)
        return DeterministicActorCritic(actor=self._actor(rep), critic=critic).to(self.device)

    def exploration(self, pi_actions, noise=None):
        """core/off_policy.py:142-144: clamp(a + randn_like(a)*noise_scale, low, high), in one K8T launch."""
        a = pi_actions.to(torch.float32).contiguous()
        noise = torch.randn_like(a) if noise is None else noise.to(device=a.device, dtype=torch.float32).contiguous()
        out = torch.empty_like(a)
        B, D = a.shape
        _lib.call("xb_perturb_actions", _lib.ptr(a), _lib.ptr(noise), B, D, float(self.noise_scale), -1.0,
                  _lib.ptr(self._act_low), _lib.ptr(self._act_high), _lib.ptr(out))
        return out

    @torch.no_grad()
    def get_actions(self, observations, test_mode=False, noise=None):
        """The actor's action, plus exploration noise unless ``test_mode``.  ``noise`` (standard normal [N, action_dim])
        may be supplied for reproducible tests."""
        if isinstance(observations, np.ndarray):
            observations = torch.from_numpy(observations)
        actions = self.model.act(observations.to(self.device, torch.float32))
        if not test_mode:
            actions = self.exploration(actions, noise)
        return ActionOutput(env_actions=actions.cpu().numpy())


class TD3_Agent(DDPG_Agent):
    def _build_model(self):
        rep = self._build_representation(self.config.representation, self.observation_space, self.config)
        critic = TwinActionValueCritic(representation=deepcopy(rep), action_space=self.action_space,
                                       critic_hidden_size=self.config.critic_hidden_size, normalizer=self.normalize_fn,
                                       initializer=self.initializer, activation=self.activation, device=self.device)
        return TwinDelayedActorCritic(actor=self._actor(rep), critic=critic,
                                      target_policy_noise=getattr(self.config, "target_policy_noise", 0.2),
                                      target_noise_clip=getattr(self.config, "target_noise_clip", 0.5)).to(self.device)

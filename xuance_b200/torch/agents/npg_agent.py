"""Natural policy gradient agent - mirror of xuance/torch/agents/policy_gradient/npg_agent.py:15-67.

The model is the reference's: a CategoricalActor (Discrete) or GaussianActor (Box) on the representation and a
StateValueCritic on a deep copy of it, in an ActorCritic.  Acting and the rollout loops (host and ``device_rollout``) are
PPO_Agent's, through K10 / K10G on the actor's raw outputs.  The buffer keeps PPO_Agent's ``old_logp`` field, which the
device rollout writes K10's log-probabilities into; the NPG update does not read it."""
from copy import deepcopy

from ...common.spaces import is_discrete
from ..rl_models import GaussianActor, CategoricalActor, StateValueCritic, ActorCritic, ActivationFunctions
from .ppo_agent import PPO_Agent

MAX_ACTIONS = 64        # K4N: A <= 64 actions, D <= 64 action components


class NPG_Agent(PPO_Agent):
    def _build_model(self):
        """npg_agent.py:37-67."""
        if self.use_actions_mask:
            raise NotImplementedError("NPG with action masks is not supported")
        if self.world_size > 1:
            raise NotImplementedError("NPG runs on one GPU: multi-GPU training is not supported")
        gaussian = self._gaussian_policy
        if not (is_discrete(self.action_space) or gaussian):
            raise NotImplementedError("NPG supports Discrete and one-dimensional Box action spaces, got %r"
                                      % (self.action_space,))
        n = self.action_space.shape[0] if gaussian else self.action_space.n
        if n > MAX_ACTIONS:
            raise NotImplementedError("NPG: the fused loss takes at most %d %s, this space has %d"
                                      % (MAX_ACTIONS, "action components" if gaussian else "actions", n))
        rep = self._build_representation(self.config.representation, self.observation_space, self.config)
        kw = dict(normalizer=self.normalize_fn, initializer=self.initializer, activation=self.activation,
                  device=self.device)
        if gaussian:
            actor = GaussianActor(representation=rep, actor_hidden_size=self.config.actor_hidden_size,
                                  action_space=self.action_space,
                                  activation_action=ActivationFunctions[self.config.activation_action], **kw)
        else:
            actor = CategoricalActor(representation=rep, actor_hidden_size=self.config.actor_hidden_size,
                                     action_space=self.action_space, **kw)
        critic = StateValueCritic(representation=deepcopy(rep), critic_hidden_size=self.config.critic_hidden_size, **kw)
        return ActorCritic(actor=actor, critic=critic).to(self.device)

"""Phasic Policy Gradient agent - mirror of xuance/torch/agents/policy_gradient/ppg_agent.py:20-248.

Acting and the rollout loops (host and ``device_rollout``) are PPO_Agent's: the actor's raw outputs go through K10 /
K10G, and the buffer stores the acting-time ``old_logp`` that the policy phase's PPO-Clip surrogate needs.  The update
cycle (``train_epochs``, run when the buffer is full) is the reference's three phases plus the relabel between the
second and the third (ppg_agent.py:155-203).

Differences in the random stream only: the reference's relabel calls ``get_actions`` over the whole buffer, which draws
(and discards) N*T action samples from torch's generator; here the relabel is one no-grad actor forward that draws
nothing.  The ``old_dist`` rows of the buffer are written only by the relabel: before it they hold whatever the
previous cycle left, and nothing reads them then."""
from copy import deepcopy

import numpy as np
import torch

from ...common.spaces import is_discrete
from ..rl_models import GaussianActor, CategoricalActor, StateValueCritic, PhasicActorCritic, ActivationFunctions
from .ppo_agent import PPO_Agent

MAX_ACTIONS = 64        # K4 / K4P: A <= 64 actions; K4G / K4P: D <= 64 action components


class PPG_Agent(PPO_Agent):
    def __init__(self, config, envs=None, observation_space=None, action_space=None, callback=None):
        super().__init__(config, envs, observation_space, action_space, callback)    # PPG_Learner refuses world_size > 1
        self.policy_nepoch = config.policy_nepoch
        self.value_nepoch = config.value_nepoch
        self.aux_nepoch = config.aux_nepoch

    def _build_model(self):
        """ppg_agent.py:47-93: an actor on the representation and two StateValueCritics on deep copies of it."""
        if self.use_actions_mask:
            raise NotImplementedError("PPG with action masks is not supported")
        gaussian = self._gaussian_policy
        if not (is_discrete(self.action_space) or gaussian):
            raise NotImplementedError("PPG supports Discrete and one-dimensional Box action spaces, got %r"
                                      % (self.action_space,))
        n = self.action_space.shape[0] if gaussian else self.action_space.n
        if n > MAX_ACTIONS:
            raise NotImplementedError("PPG: the fused losses take at most %d %s, this space has %d"
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
        aux_critic = StateValueCritic(representation=deepcopy(rep), critic_hidden_size=self.config.critic_hidden_size,
                                      **kw)
        return PhasicActorCritic(actor=actor, critic=critic, aux_critic=aux_critic).to(self.device)

    @property
    def auxiliary_info_shape(self):
        """``old_logp`` from acting (the policy phase), ``old_dist`` = the relabelled actor's raw logits (Discrete) or
        means (Box) per slot (the auxiliary phase)."""
        k = self.action_space.shape[0] if self._gaussian_policy else self.action_space.n
        return {"old_logp": (), "old_dist": (k,)}

    @torch.no_grad()
    def _relabel(self):
        """ppg_agent.py:186-191: the current actor over every observation of the buffer, written straight into the
        buffer's ``old_dist`` rows (and, for a Box space, the log_std snapshot)."""
        mem = self.memory
        rows = mem.aux_rows["old_dist"]
        obs = mem.observations.reshape((-1,) + tuple(mem.observations.shape[2:]))
        if self._gaussian_policy:
            mu, log_std = self.model.mu_log_std(obs)
            rows.copy_(mu.reshape(rows.shape))
            mem.dist_log_std.copy_(log_std)
        else:
            rows.copy_(self.model.logits(obs).reshape(rows.shape))

    def _phase(self, update, n_epochs, indexes):
        """``n_epochs`` x minibatches of ``update``; ``indexes`` is shuffled in place before every epoch, as the one
        array the reference shares across the phases.  Only the phase's last minibatch reads its statistics."""
        info = {}
        total, done = n_epochs * -(-self.buffer_size // self.batch_size), 0
        for _ in range(n_epochs):
            np.random.shuffle(indexes)
            perm_d = torch.from_numpy(indexes).to(self.device)     # one H2D per epoch
            for start in range(0, self.buffer_size, self.batch_size):
                done += 1
                samples = self.memory.sample(perm_d[start:start + self.batch_size])
                info = update(sync=(done == total), **samples)
        return info

    def train_epochs(self, n_epochs=1):
        """One PPG update cycle (ppg_agent.py:163-201): policy phase, critic phase, relabel, auxiliary phase.  The
        phases' epoch counts are ``policy_nepoch`` / ``value_nepoch`` / ``aux_nepoch``; ``n_epochs`` is not used, as in
        the reference.  Returns the last minibatch's info of each phase, merged."""
        self.memory._ensure_gae()
        indexes = np.arange(self.buffer_size)
        info = {}
        info.update(self._phase(self.learner.update_actor, self.policy_nepoch, indexes))
        info.update(self._phase(self.learner.update_critic, self.value_nepoch, indexes))
        self._relabel()
        info.update(self._phase(self.learner.update_auxiliary_critic, self.aux_nepoch, indexes))
        return info

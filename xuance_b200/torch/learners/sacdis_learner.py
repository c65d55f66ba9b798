"""SAC-Discrete learner - mirror of xuance/torch/learners/policy_gradient/sacdis_learner.py:12-129.

Same three optimiser steps in the same order (actor, critic, temperature), the same LinearLR schedules, soft target update
and info keys as the reference.  The probability / log rules, both losses and their backward seeds are the K8D kernels;
each optimiser is a flat-bucket K7 Adam (actor bucket, critic bucket, log_alpha), and the Polyak update streams over the
critic / target-critic buckets once (K7 xb_soft_update).  alpha never leaves the device.  Everything but the actor and
critic steps and the target entropy is SAC's (sac_learner._SoftActorCritic_Learner).

One critic forward on ``obs`` serves both steps: the actor step does not change the critic, and the actor's gradient to
the critic's outputs is not needed (the reference's critic.zero_grad() discards it).  The target runs after the actor's
Adam step, as the reference's Qtarget does."""
import torch

from ... import _lib
from .sac_learner import _SoftActorCritic_Learner


class SACDIS_Learner(_SoftActorCritic_Learner):
    def __init__(self, config, model, callback):
        self.n_actions = int(model.actor.action_dim)
        super().__init__(config, model, callback)

    def _target_entropy(self):
        # the reference reads model.action_space.n, an attribute SoftActorCriticDiscrete lacks (it raises
        # AttributeError there); its evident intent is -A (DESIGN.md section 4)
        return -float(self.n_actions)

    def _graph_key_and_args(self, args, samples):
        return tuple(args[0].shape), args

    def _actor_critic_steps(self, obs, act, nxt, rew, ter):
        """sacdis_learner.py:52-75 on the device."""
        B, A = obs.shape[0], self.n_actions
        Bt = B * self.world_size
        alpha = self._alpha_buf

        # ---- actor step (sacdis_learner.py:52-60); q1 / q2 keep their graph for the critic step
        logits, q1, q2 = self.model.Qpolicy(obs)
        dlogits = torch.empty_like(logits)
        _lib.call("xb_sacdis_actor_loss", _lib.ptr(logits), _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(alpha), B, A, Bt,
                  _lib.ptr(dlogits), _lib.ptr(self._stats_a), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer['actor'], [logits], [dlogits], inputs=self.optimizer['actor'].bucket.params)

        # ---- critic step (:62-75) with the just-updated actor on obs_next
        with torch.no_grad():
            logits_next, tq1, tq2 = self.model.Qtarget(nxt)
        dq1, dq2, backup = torch.empty_like(q1), torch.empty_like(q2), torch.empty_like(rew)
        _lib.call("xb_sacdis_critic_loss", _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(act), _lib.ptr(logits_next),
                  _lib.ptr(tq1), _lib.ptr(tq2), _lib.ptr(rew), _lib.ptr(ter), _lib.ptr(alpha), float(self.gamma), B, A,
                  Bt, _lib.ptr(dq1), _lib.ptr(dq2), _lib.ptr(backup), _lib.ptr(self._stats_c), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer['critic'], [q1, q2], [dq1, dq2], inputs=self.optimizer['critic'].bucket.params)

"""DDPG and TD3 learners - mirror of xuance/torch/learners/policy_gradient/ddpg_learner.py:12-94 and
td3_learner.py:12-100.

The same optimiser steps in the same order, the same LinearLR schedules, soft target updates and info keys.  The elementwise
loss stages and their backward seeds are the K8T kernels, each optimiser is a flat-bucket K7 Adam (actor bucket, critic
bucket), and the Polyak update streams over the flat target buckets (two K7 xb_soft_update launches).  No host
synchronisation happens before the info dict is built.

* DDPG, every iteration: critic step, actor step on the UPDATED critic, both schedulers, soft update of both targets.
* TD3, every iteration: critic step (on smoothed target actions), the critic scheduler; every ``actor_update_delay``-th
  iteration also: actor step, the actor scheduler, soft update.  The actor's Adam step count advances only then.

One collective per optimiser step, critic then actor (they cannot merge: the actor step reads the updated critic)."""
import torch

from ... import _lib
from .sac_learner import _ActorCritic_Learner


class DDPG_Learner(_ActorCritic_Learner):
    twin = False
    target_names = ('actor', 'critic')

    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        self.actor_update_delay = getattr(config, "actor_update_delay") if self.twin else 1
        # the logged statistics ride in the tails of the two gradient buckets (the same collective as the gradient)
        self._stats_a = self.optimizer['actor'].bucket.tail[:4]
        self._stats_c = self.optimizer['critic'].bucket.tail[:4]
        self._scratch = _lib.scratch(self.device)

    @staticmethod
    def _flat(x):
        return None if x is None else x.reshape(-1).contiguous()

    def _device_update(self, obs, act, nxt, rew, ter, actor_step, noise_next=None):
        """Everything of one update that runs on the device; static shapes, no host synchronisation."""
        B = obs.shape[0]
        Bt = B * self.world_size
        P, F = _lib.ptr, self._flat

        # ---- critic step (ddpg_learner.py:45-54, td3_learner.py:46-59)
        q = self.model.Qaction(obs, act)
        q1, q2 = (F(q[0]), F(q[1])) if self.twin else (F(q), None)
        with torch.no_grad():
            tq1, tq2 = self.model.Qtarget_pair(nxt, noise_next) if self.twin else self.model.Qtarget_pair(nxt)
            tq1, tq2 = F(tq1), F(tq2)
        dq1, dq2, backup = torch.empty_like(q1), (None if q2 is None else torch.empty_like(q2)), torch.empty_like(q1)
        _lib.call("xb_ddpg_critic_loss", P(q1), P(q2), P(tq1), P(tq2), P(rew), P(ter), float(self.gamma), B, Bt, P(dq1),
                  P(dq2), P(backup), P(self._stats_c), P(self._scratch))
        outs, grads = ([q1, q2], [dq1, dq2]) if self.twin else ([q1], [dq1])
        self._optimizer_step(self.optimizer['critic'], outs, grads)

        # ---- actor step on the updated critic (ddpg_learner.py:56-63, td3_learner.py:63-73)
        if actor_step:
            p1, p2 = self.model.Qpolicy_pair(obs)
            p1, p2 = F(p1), F(p2)
            dp1, dp2 = torch.empty_like(p1), (None if p2 is None else torch.empty_like(p2))
            _lib.call("xb_ddpg_actor_loss", P(p1), P(p2), B, Bt, P(dp1), P(dp2), P(self._stats_a), P(self._scratch))
            outs, grads = ([p1, p2], [dp1, dp2]) if self.twin else ([p1], [dp1])
            # the reference's p_loss.backward() also fills the critic's gradients; its next zero_grad discards them
            self._optimizer_step(self.optimizer['actor'], outs, grads, inputs=self.optimizer['actor'].bucket.params)
            self._soft_update()
        return None

    def update(self, sync=True, noise_next=None, **samples):
        """``noise_next`` (standard normal [B, action_dim], TD3 only) may be supplied for reproducible tests; by default
        the model draws it with torch.randn_like, as the reference does."""
        self.iterations += 1
        actor_step = self.iterations % self.actor_update_delay == 0
        obs, act = self._f32(samples['obs']), self._f32(samples['actions'])
        nxt, rew, ter = self._f32(samples['obs_next']), self._f32(samples['rewards']), self._f32(samples['terminals'])
        info = self.callback.on_update_start(self.iterations, model=self.model, obs=obs, act=act, next_obs=nxt,
                                             rew=rew, termination=ter) or {}
        self.optimizer['critic'].prepare()
        if actor_step:
            self.optimizer['actor'].prepare()
        noise = None if noise_next is None or not self.twin else self._f32(noise_next)
        args = [obs, act, nxt, rew, ter] + ([] if noise is None else [noise])
        self._device_step((tuple(obs.shape), actor_step, len(args)),
                          lambda *a: self._device_update(*a[:5], actor_step, *a[5:]), *args)
        self.scheduler['critic'].step()
        if actor_step:
            self.scheduler['actor'].step()
        if sync:
            sc = self._stats_c.tolist()
            vals = {"Qloss": sc[0]}
            if actor_step:
                vals["Ploss"] = self._stats_a[0].item()
            if self.twin:
                vals.update(QvalueA=sc[1], QvalueB=sc[2])
            else:
                vals["Qvalue"] = sc[1]
            vals.update(actor_lr=self.optimizer['actor'].param_groups[0]['lr'],
                        critic_lr=self.optimizer['critic'].param_groups[0]['lr'])
            self._finish_info(info, vals, model=self.model)
        return info


class TD3_Learner(DDPG_Learner):
    twin = True

"""Soft Actor-Critic learner - mirror of xuance/torch/learners/policy_gradient/sac_learner.py:13-126.

Same three optimiser steps in the same order (actor, critic, alpha), the same LinearLR schedules, soft target
update and info keys.  The elementwise loss stages and their backward seeds are the K8 kernels, each optimiser is
a flat-bucket K7 Adam (actor bucket, critic bucket, log_alpha), the Polyak update streams over the critic /
target-critic buckets once (K7 xb_soft_update).  alpha never leaves the device.

``_SoftActorCritic_Learner`` holds what SAC and SAC-Discrete (sacdis_learner.py) share: the optimisers, the target
critic, the temperature state and step, ``update`` and the info dict.  ``_ActorCritic_Learner`` holds the actor / critic
optimisers and the target buckets that DDPG and TD3 (ddpg_learner.py) share with them."""
import numpy as np
import torch
import torch.nn as nn

from ... import _lib
from ..utils import FusedAdam
from ..utils.flat_bucket import target_bucket
from .learner import Learner


class _ActorCritic_Learner(Learner):
    """An actor and a critic, each with its own FusedAdam and LinearLR, and a target copy of each network named in
    ``target_names``, held in a flat array laid out as the live network's bucket."""
    target_names = ('critic',)

    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        self.optimizer = {
            'actor': FusedAdam(self.model.actor.parameters(), self.config.learning_rate_actor),
            'critic': FusedAdam(self.model.critic.parameters(), self.config.learning_rate_critic)}
        self.scheduler = {k: self._linear_lr(o) for k, o in self.optimizer.items()}
        self._targets = {k: target_bucket(getattr(self.model, "target_" + k), self.optimizer[k].bucket)
                         for k in self.target_names}
        self._graph_tensors = [t.flat for t in self._targets.values()]
        self.tau, self.gamma = config.tau, config.gamma

    def _soft_update(self):
        """Polyak update of every target (actor_critic.py:155-158, 255-261, 313-319): one K7 launch per target."""
        for k, tgt in self._targets.items():
            live = self.optimizer[k].bucket
            _lib.call("xb_soft_update", _lib.ptr(tgt.flat), _lib.ptr(live.flat), live.numel, float(self.tau))


class _SoftActorCritic_Learner(_ActorCritic_Learner):
    """Subclasses supply ``_actor_critic_steps`` (the actor step, then the critic step), ``_target_entropy`` and
    ``_graph_key_and_args``."""

    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        self.use_automatic_entropy_tuning = config.use_automatic_entropy_tuning
        if self.use_automatic_entropy_tuning:
            self.target_entropy = self._target_entropy()
            self.log_alpha = nn.Parameter(torch.zeros(1, requires_grad=True, device=self.device))
            self.alpha_optimizer = FusedAdam([self.log_alpha], lr=config.learning_rate_actor)
            self._alpha_buf = self.log_alpha.detach().exp()
        else:
            self._alpha_buf = torch.full((1,), float(config.alpha), device=self.device)
        self.alpha = self._alpha_buf
        self._graph_tensors.append(self._alpha_buf)
        # the logged sums (and mean(log_pi), which the temperature step needs globally) ride in the tails of the two gradient
        # buckets: TWO collectives per update.  They cannot be one: the reference steps the actor before it evaluates the
        # critic target (sac_learner.py:53-72), so the critic gradient does not exist when the actor's must be reduced.
        self._stats_a = self.optimizer['actor'].bucket.tail[:4]
        self._stats_c = self.optimizer['critic'].bucket.tail[:2]
        self._scratch = _lib.scratch(self.device)
        self._alpha_loss = torch.zeros(1, dtype=torch.float32, device=self.device)

    def _optimizers(self):
        # the temperature optimiser is stepped with the others but, as in the reference, not checkpointed
        return super()._optimizers() + ([self.alpha_optimizer] if self.use_automatic_entropy_tuning else [])

    def _device_update(self, *args):
        """Everything of one update that runs on the device; no host synchronisation, static shapes."""
        self._actor_critic_steps(*args)
        # ---- temperature step (sac_learner.py:74-82, sacdis_learner.py:77-86): d/dlog_alpha of
        # -mean(log_alpha * (log_pi + H_target)) = -(mean(log_pi) + H_target)
        if self.use_automatic_entropy_tuning:
            g = -(self._stats_a[2:3] + self.target_entropy)      # already the global mean: summed with the actor gradient
            self._alpha_loss.copy_(self.log_alpha.detach() * g)
            self.alpha_optimizer.zero_grad()
            self.alpha_optimizer.bucket.grad[:1].copy_(g)
            self.alpha_optimizer.launch()
            torch.exp(self.log_alpha.detach(), out=self._alpha_buf)
        self._soft_update()
        return None

    def update(self, sync=True, **samples):
        self.iterations += 1
        obs, act = self._f32(samples['obs']), self._f32(samples['actions'])
        nxt, rew, ter = self._f32(samples['obs_next']), self._f32(samples['rewards']), self._f32(samples['terminals'])
        info = self.callback.on_update_start(self.iterations, model=self.model, obs=obs, act=act, next_obs=nxt,
                                             rew=rew, termination=ter) or {}
        for o in self.optimizer.values():
            o.prepare()
        if self.use_automatic_entropy_tuning:
            self.alpha_optimizer.prepare()
        key, args = self._graph_key_and_args([obs, act, nxt, rew, ter], samples)
        self._device_step(key, self._device_update, *args)
        self.alpha = self._alpha_buf
        for sch in self.scheduler.values():
            sch.step()
        if sync:
            sa, sc = self._stats_a.tolist(), self._stats_c.tolist()
            vals = {"Qloss": sc[0], "Ploss": sa[0], "Qvalue": sa[1],
                    "actor_lr": self.optimizer['actor'].param_groups[0]['lr'],
                    "critic_lr": self.optimizer['critic'].param_groups[0]['lr']}
            if self.use_automatic_entropy_tuning:
                vals.update(alpha_loss=float(self._alpha_loss), alpha=float(self._alpha_buf))
            self._finish_info(info, vals, model=self.model)
        return info


class SAC_Learner(_SoftActorCritic_Learner):
    def _target_entropy(self):
        return -np.prod(self.model.actor.action_space.shape).item()

    def _graph_key_and_args(self, args, samples):
        """``noise_pi`` / ``noise_next`` (standard normal [B, act_dim]) may be supplied for reproducible tests; by default
        the model draws them as the reference does (Normal.rsample).  With only one of them the update runs eagerly."""
        noise_pi, noise_next = samples.get('noise_pi'), samples.get('noise_next')
        if noise_pi is not None or noise_next is not None:
            args = args + [noise_pi, noise_next]
        graphed = (noise_pi is None) == (noise_next is None)
        return ((tuple(args[0].shape), len(args)) if graphed else None), args

    def _actor_critic_steps(self, obs, act, nxt, rew, ter, noise_pi=None, noise_next=None):
        """sac_learner.py:52-72 on the device."""
        B = obs.shape[0]
        Bt = B * self.world_size
        alpha = self._alpha_buf

        # ---- actor step (sac_learner.py:53-60)
        log_pi, q1, q2 = self.model.Qpolicy(obs, noise_pi)
        log_pi, q1, q2 = log_pi.reshape(-1).contiguous(), q1.reshape(-1).contiguous(), q2.reshape(-1).contiguous()
        dlp, dq1, dq2 = torch.empty_like(log_pi), torch.empty_like(q1), torch.empty_like(q2)
        _lib.call("xb_sac_actor_loss", _lib.ptr(log_pi), _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(alpha), B, Bt,
                  _lib.ptr(dlp), _lib.ptr(dq1), _lib.ptr(dq2), _lib.ptr(self._stats_a), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer['actor'], [log_pi, q1, q2], [dlp, dq1, dq2],
                             inputs=self.optimizer['actor'].bucket.params)

        # ---- critic step (:62-72)
        aq1, aq2 = self.model.Qaction(obs, act)
        aq1, aq2 = aq1.reshape(-1).contiguous(), aq2.reshape(-1).contiguous()
        with torch.no_grad():
            log_pi_next, target_q = self.model.Qtarget(nxt, noise_next)
            log_pi_next, target_q = log_pi_next.reshape(-1).contiguous(), target_q.reshape(-1).contiguous()
        dq1, dq2, backup = torch.empty_like(aq1), torch.empty_like(aq2), torch.empty_like(aq1)
        _lib.call("xb_sac_critic_loss", _lib.ptr(aq1), _lib.ptr(aq2), _lib.ptr(target_q), _lib.ptr(log_pi_next),
                  _lib.ptr(rew), _lib.ptr(ter), _lib.ptr(alpha), float(self.gamma), B, Bt, _lib.ptr(dq1), _lib.ptr(dq2),
                  _lib.ptr(backup), _lib.ptr(self._stats_c), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer['critic'], [aq1, aq2], [dq1, dq2])

"""SAC-Discrete learner - mirror of xuance/torch/learners/policy_gradient/sacdis_learner.py:12-129.

Same three optimiser steps in the same order (actor, critic, temperature), the same LinearLR schedules, soft target update
and info keys as the reference.  The probability / log rules, both losses and their backward seeds are the K8D kernels;
each optimiser is a flat-bucket K7 Adam (actor bucket, critic bucket, log_alpha), and the Polyak update streams over the
critic / target-critic buckets once (K7 xb_soft_update).  alpha never leaves the device.

One critic forward on ``obs`` serves both steps: the actor step does not change the critic, and the actor's gradient to
the critic's outputs is not needed (the reference's critic.zero_grad() discards it).  The target runs after the actor's
Adam step, as the reference's Qtarget does."""
import torch
import torch.nn as nn

from ... import _lib
from ..utils import FusedAdam, FlatBucket, allreduce_sum_, CapturedStep
from .learner import Learner


class SACDIS_Learner(Learner):
    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        self.optimizer = {
            'actor': FusedAdam(self.model.actor.parameters(), self.config.learning_rate_actor),
            'critic': FusedAdam(self.model.critic.parameters(), self.config.learning_rate_critic)}
        mk = lambda o: torch.optim.lr_scheduler.LinearLR(o, start_factor=1.0, end_factor=self.end_factor_lr_decay,
                                                         total_iters=self.total_iters)
        self.scheduler = {'actor': mk(self.optimizer['actor']), 'critic': mk(self.optimizer['critic'])}
        self._target_bucket = FlatBucket([p.requires_grad_(True) for p in self.model.target_critic.parameters()])
        for p in self.model.target_critic.parameters():
            p.requires_grad_(False)
            p.grad = None
        assert self._target_bucket.numel == self.optimizer['critic'].bucket.numel
        self.n_actions = int(self.model.actor.action_dim)
        self.tau, self.gamma = config.tau, config.gamma
        self.use_automatic_entropy_tuning = config.use_automatic_entropy_tuning
        if self.use_automatic_entropy_tuning:
            # the reference reads model.action_space.n, an attribute SoftActorCriticDiscrete lacks (it raises
            # AttributeError there); its evident intent is -A (DESIGN.md section 4)
            self.target_entropy = -float(self.n_actions)
            self.log_alpha = nn.Parameter(torch.zeros(1, requires_grad=True, device=self.device))
            self.alpha_optimizer = FusedAdam([self.log_alpha], lr=config.learning_rate_actor)
            self._alpha_buf = self.log_alpha.detach().exp()
        else:
            self._alpha_buf = torch.full((1,), float(config.alpha), device=self.device)
        self.alpha = self._alpha_buf
        self.use_cuda_graph = getattr(config, "use_cuda_graph", False)
        self._graphs = {}
        # the logged sums (and mean(log_pi), which the temperature step needs globally) ride in the tails of the two
        # gradient buckets: TWO collectives per update, for SAC's reason - the critic target needs the updated actor
        self._stats_a = self.optimizer['actor'].bucket.tail[:4]
        self._stats_c = self.optimizer['critic'].bucket.tail[:2]
        self._scratch = _lib.scratch(self.device)
        self._alpha_loss = torch.zeros(1, dtype=torch.float32, device=self.device)

    def _f32(self, x):
        return torch.as_tensor(x, device=self.device).to(torch.float32).contiguous()

    def _snapshot(self):
        st = {k: v.snapshot() for k, v in self.optimizer.items()}
        st["target"] = self._target_bucket.flat.clone()
        if self.use_automatic_entropy_tuning:
            st["alpha_opt"] = self.alpha_optimizer.snapshot()
        st["alpha"] = self._alpha_buf.clone()
        return st

    def _restore(self, st):
        for k, v in self.optimizer.items():
            v.restore(st[k])
        self._target_bucket.flat.copy_(st["target"])
        if self.use_automatic_entropy_tuning:
            self.alpha_optimizer.restore(st["alpha_opt"])
        self._alpha_buf.copy_(st["alpha"])

    def _device_update(self, obs, act, nxt, rew, ter):
        """Everything of sacdis_learner.py:52-91 that runs on the device; no host synchronisation, static shapes."""
        B, A = obs.shape[0], self.n_actions
        Bt = B * self.world_size
        clip = self.grad_clip_norm if self.use_grad_clip else None
        alpha = self._alpha_buf

        # ---- actor step (sacdis_learner.py:52-60); q1 / q2 keep their graph for the critic step
        logits, q1, q2 = self.model.Qpolicy(obs)
        dlogits = torch.empty_like(logits)
        _lib.call("xb_sacdis_actor_loss", _lib.ptr(logits), _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(alpha), B, A, Bt,
                  _lib.ptr(dlogits), _lib.ptr(self._stats_a), _lib.ptr(self._scratch))
        self.optimizer['actor'].zero_grad()
        torch.autograd.backward([logits], [dlogits], inputs=self.optimizer['actor'].bucket.params)
        if self.world_size > 1:
            allreduce_sum_(self.optimizer['actor'].bucket.grad_all)
        self.optimizer['actor'].launch(max_norm=clip)

        # ---- critic step (:62-75) with the just-updated actor on obs_next
        with torch.no_grad():
            logits_next, tq1, tq2 = self.model.Qtarget(nxt)
        dq1, dq2, backup = torch.empty_like(q1), torch.empty_like(q2), torch.empty_like(rew)
        _lib.call("xb_sacdis_critic_loss", _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(act), _lib.ptr(logits_next),
                  _lib.ptr(tq1), _lib.ptr(tq2), _lib.ptr(rew), _lib.ptr(ter), _lib.ptr(alpha), float(self.gamma), B, A,
                  Bt, _lib.ptr(dq1), _lib.ptr(dq2), _lib.ptr(backup), _lib.ptr(self._stats_c), _lib.ptr(self._scratch))
        self.optimizer['critic'].zero_grad()
        torch.autograd.backward([q1, q2], [dq1, dq2], inputs=self.optimizer['critic'].bucket.params)
        if self.world_size > 1:
            allreduce_sum_(self.optimizer['critic'].bucket.grad_all)
        self.optimizer['critic'].launch(max_norm=clip)

        # ---- temperature step (:77-86): d/dlog_alpha of -mean(log_alpha*(log_pi + H_target)) over all B*A entries of
        # the unweighted log_pi matrix = -(mean(log_pi) + H_target)
        if self.use_automatic_entropy_tuning:
            g = -(self._stats_a[2:3] + self.target_entropy)      # already the global mean: summed with the actor gradient
            self._alpha_loss.copy_(self.log_alpha.detach() * g)
            self.alpha_optimizer.zero_grad()
            self.alpha_optimizer.bucket.grad[:1].copy_(g)
            self.alpha_optimizer.launch()
            torch.exp(self.log_alpha.detach(), out=self._alpha_buf)

        cb = self.optimizer['critic'].bucket
        _lib.call("xb_soft_update", _lib.ptr(self._target_bucket.flat), _lib.ptr(cb.flat), cb.numel, float(self.tau))
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
        if self.use_cuda_graph:
            args = [obs, act, nxt, rew, ter]
            key = tuple(obs.shape)
            if key not in self._graphs:
                self._graphs[key] = CapturedStep(self._device_update, args, self._snapshot, self._restore)
            self._graphs[key](*args)
        else:
            self._device_update(obs, act, nxt, rew, ter)
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
            if self.distributed_training:
                vals = {f"{k}/rank_{self.rank}": v for k, v in vals.items()}
            info.update(vals)
            info.update(self.callback.on_update_end(self.iterations, model=self.model, info=info) or {})
        return info

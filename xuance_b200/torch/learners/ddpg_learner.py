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
from ..utils import FusedAdam, FlatBucket, allreduce_sum_, CapturedStep
from .learner import Learner


def _target_bucket(target, live_bucket):
    """The target network's parameters in their own flat array, in the live bucket's parameter order and layout."""
    params = list(target.parameters())
    bucket = FlatBucket([p.requires_grad_(True) for p in params])
    for p in params:
        p.requires_grad_(False)
        p.grad = None
    assert bucket.numel == live_bucket.numel and bucket.offsets == live_bucket.offsets
    return bucket


class DDPG_Learner(Learner):
    twin = False

    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        self.optimizer = {
            'actor': FusedAdam(self.model.actor.parameters(), self.config.learning_rate_actor),
            'critic': FusedAdam(self.model.critic.parameters(), self.config.learning_rate_critic)}
        mk = lambda o: torch.optim.lr_scheduler.LinearLR(o, start_factor=1.0, end_factor=self.end_factor_lr_decay,
                                                         total_iters=self.total_iters)
        self.scheduler = {'actor': mk(self.optimizer['actor']), 'critic': mk(self.optimizer['critic'])}
        self._targets = {'actor': _target_bucket(self.model.target_actor, self.optimizer['actor'].bucket),
                         'critic': _target_bucket(self.model.target_critic, self.optimizer['critic'].bucket)}
        self.tau, self.gamma = config.tau, config.gamma
        self.actor_update_delay = getattr(config, "actor_update_delay") if self.twin else 1
        self.use_cuda_graph = getattr(config, "use_cuda_graph", False)
        self._graphs = {}
        # the logged statistics ride in the tails of the two gradient buckets (the same collective as the gradient)
        self._stats_a = self.optimizer['actor'].bucket.tail[:4]
        self._stats_c = self.optimizer['critic'].bucket.tail[:4]
        self._scratch = _lib.scratch(self.device)

    def _f32(self, x):
        return torch.as_tensor(x, device=self.device).to(torch.float32).contiguous()

    def _snapshot(self):
        st = {k: v.snapshot() for k, v in self.optimizer.items()}
        st.update({"target_" + k: v.flat.clone() for k, v in self._targets.items()})
        return st

    def _restore(self, st):
        for k, v in self.optimizer.items():
            v.restore(st[k])
        for k, v in self._targets.items():
            v.flat.copy_(st["target_" + k])

    @staticmethod
    def _flat(x):
        return None if x is None else x.reshape(-1).contiguous()

    def _step(self, name, outputs, grads, clip, inputs=None):
        opt = self.optimizer[name]
        opt.zero_grad()
        torch.autograd.backward(outputs, grads, inputs=inputs)
        if self.world_size > 1:
            allreduce_sum_(opt.bucket.grad_all)
        opt.launch(max_norm=clip)

    def _device_update(self, obs, act, nxt, rew, ter, actor_step, noise_next=None):
        """Everything of one update that runs on the device; static shapes, no host synchronisation."""
        B = obs.shape[0]
        Bt = B * self.world_size
        clip = self.grad_clip_norm if self.use_grad_clip else None
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
        self._step('critic', outs, grads, clip)

        # ---- actor step on the updated critic (ddpg_learner.py:56-63, td3_learner.py:63-73)
        if actor_step:
            p1, p2 = self.model.Qpolicy_pair(obs)
            p1, p2 = F(p1), F(p2)
            dp1, dp2 = torch.empty_like(p1), (None if p2 is None else torch.empty_like(p2))
            _lib.call("xb_ddpg_actor_loss", P(p1), P(p2), B, Bt, P(dp1), P(dp2), P(self._stats_a), P(self._scratch))
            outs, grads = ([p1, p2], [dp1, dp2]) if self.twin else ([p1], [dp1])
            # the reference's p_loss.backward() also fills the critic's gradients; its next zero_grad discards them
            self._step('actor', outs, grads, clip, inputs=self.optimizer['actor'].bucket.params)
            # ---- Polyak update of both targets (actor_critic.py:255-261, 313-319)
            for k, tgt in self._targets.items():
                live = self.optimizer[k].bucket
                _lib.call("xb_soft_update", P(tgt.flat), P(live.flat), live.numel, float(self.tau))
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
        if self.use_cuda_graph:
            key = (tuple(obs.shape), actor_step, len(args))
            if key not in self._graphs:
                fn = lambda *a, s=actor_step: self._device_update(*a[:5], s, *a[5:])
                self._graphs[key] = CapturedStep(fn, args, self._snapshot, self._restore)
            self._graphs[key](*args)
        else:
            self._device_update(*args[:5], actor_step, *args[5:])
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
            if self.distributed_training:
                vals = {f"{k}/rank_{self.rank}": v for k, v in vals.items()}
            info.update(vals)
            info.update(self.callback.on_update_end(self.iterations, model=self.model, info=info) or {})
        return info


class TD3_Learner(DDPG_Learner):
    twin = True

"""COMA learner - mirror of xuance/torch/learners/multi_agent_rl/coma_learner.py:14-153 (on IAC_Learner) for one
parameter-sharing group with Discrete actions.

update(sample, epsilon): actor logits and the live critics' Q over the packed (b, i, t) rows (the critic input assembled by
K4C) -> ``xb_mappo_prepare`` (global mask sum) -> [all-reduce of that block] -> K4C fused loss forward + backward
(dlogits, dQ, statistics into the critic bucket's tail) -> the critic's backward and K7 clip + Adam, then the actor's.
Epsilon lives in a device scalar, so the device half is capturable as one CUDA graph (``use_cuda_graph``) whose replays
follow the decaying epsilon.  The target sync (``iterations % sync_frequency == 0``) and both LinearLR steps run on the
host after the device half; the actor step does not read the critics, so this equals the reference's order (critic
step, sync, actor step)."""
import torch

from ... import _lib
from ..utils import FusedAdam, allreduce_sum_
from .vdac_learner import IAC_Learner


class COMA_Learner(IAC_Learner):
    def __init__(self, config, agent_grouping, model, callback):
        # coma_learner.py:20-23: no value clipping, Huber loss, value normalisation or loss coefficients
        config.use_value_clip, config.value_clip_range = False, None
        config.use_huber_loss, config.huber_delta = False, None
        config.use_value_norm = False
        config.vf_coef, config.ent_coef = None, None
        super().__init__(config, agent_grouping, model, callback)
        self.use_global_state = True
        self.sync_frequency = config.sync_frequency
        self._eps = torch.zeros(1, dtype=torch.float32, device=self.device)

    def _build_optimizer(self, config):
        """coma_learner.py:29-43: Adam(eps=1e-5) for the actors and for the critics, each with a LinearLR."""
        self.optimizer = {'actor': FusedAdam(self.model.actors.parameters(), lr=config.learning_rate_actor, eps=1e-5),
                          'critic': FusedAdam(self.model.critics.parameters(), lr=config.learning_rate_critic,
                                              eps=1e-5)}
        self.scheduler = {k: self._linear_lr(v) for k, v in self.optimizer.items()}

    def _opt(self):
        return self.optimizer['critic']      # its bucket tail carries the statistics through the critic's all-reduce

    def _device_update(self, obs, actions, adv, values_old, returns, mask, avail=None, state=None):
        """coma_learner.py:63-137 on the device (static shapes, no host synchronisation).  Rows are in (b, i, t)
        order; obs is [B*n, T, obs] with use_rnn, else [B*n, obs]; state is [B*T, S]."""
        n = self.n_agents
        R = actions.shape[0]
        T = obs.shape[1] if self.use_rnn else 1
        B = R // (n * T)
        logits = self.model.logits(obs)
        A = logits.shape[-1]
        logits = logits.reshape(-1, A).contiguous()
        q = self.model.q_values(state.reshape(B, T, -1), obs, actions.reshape(B, n, T)).contiguous()
        _lib.call("xb_mappo_prepare", _lib.ptr(mask), _lib.ptr(returns), R, _lib.ptr(self._prep),
                  _lib.ptr(self._scratch))
        if self.world_size > 1:
            allreduce_sum_(self._prep)                       # the global sum of the mask
        dlogits, dq = torch.empty_like(logits), torch.empty_like(q)
        _lib.call("xb_coma_loss_fwd_bwd", _lib.ptr(logits), _lib.ptr(avail), 0 if avail is None else avail.shape[1],
                  _lib.ptr(q), _lib.ptr(actions), _lib.ptr(returns), _lib.ptr(mask), _lib.ptr(self._eps),
                  _lib.ptr(self._prep), R, A, R * self.world_size, _lib.ptr(dlogits), _lib.ptr(dq),
                  _lib.ptr(self._stats), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer['critic'], [q], [dq])
        self._optimizer_step(self.optimizer['actor'], [logits], [dlogits])
        return None

    def update(self, sample, epsilon=0.0, sync=True):
        self.iterations += 1
        args = self._args(sample)
        info = self.callback.on_update_start(self.iterations, model=self.model, batch=sample) or {}
        self._eps.fill_(float(epsilon))
        for opt in self.optimizer.values():
            opt.prepare()
        self._device_step(tuple(args[0].shape), self._device_update, *args)
        self.scheduler['critic'].step()
        if self.iterations % self.sync_frequency == 0:
            self.model.copy_target()
        self.scheduler['actor'].step()
        if sync:
            self._finish_info(info, self._info(self._stats.tolist()), model=self.model)
        return info

    def _info(self, s):
        """coma_learner.py:119-149.  The reference stores the critic's gradient norm under "gradient_norm_actor" and
        then overwrites it with the actor's, so the actor's is what it reports."""
        vals = {}
        if self.use_grad_clip:
            vals["gradient_norm_actor"] = float(self.optimizer['actor'].grad_norm.item())
        vals.update({"learning_rate_actor": self.optimizer['actor'].param_groups[0]['lr'],
                     "learning_rate_critic": self.optimizer['critic'].param_groups[0]['lr'],
                     "actor_loss": s[0], "critic_loss": s[1], "advantage": s[2]})
        return vals

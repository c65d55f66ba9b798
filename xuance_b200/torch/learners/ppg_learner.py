"""Phasic Policy Gradient learner - mirror of xuance/torch/learners/policy_gradient/ppg_learner.py:13-151.

``update_actor``, ``update_critic`` and ``update_auxiliary_critic`` keep the reference's signatures, info keys and
scheduler stepping.  Each runs as: network forward (cuBLAS via torch) -> one fused loss launch (K4 / K4G for the policy
phase, K4P for the critic and auxiliary phases) -> torch backward into the flat gradient bucket -> K7 clip + Adam over
the parameter groups the phase's loss reaches.  The reference's one ``torch.optim.Adam`` with ``zero_grad()`` setting
gradients to None steps only those groups, each with its own step count; ``SegmentedAdam`` over the bucket laid out
``[actor | critic | aux_critic]`` does the same.  The device halves are CUDA-graph capturable (``use_cuda_graph``); the
statistics are read from the device only when ``sync`` is set (the agent sets it on a phase's last minibatch)."""
import torch

from ... import _lib
from ..rl_models.heads import GaussianActorHead
from ..utils import SegmentedAdam
from .learner import Learner

ACTOR, CRITIC, AUX = 0, 1, 2        # parameter groups = SegmentedAdam segments, in bucket order


class PPG_Learner(Learner):
    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        if self.world_size > 1:
            raise NotImplementedError("PPG runs on one GPU: multi-GPU training is not supported")
        self.optimizer = SegmentedAdam([list(model.actor.parameters()), list(model.critic.parameters()),
                                        list(model.aux_critic.parameters())], self.config.learning_rate, eps=1e-5)
        self.scheduler = self._linear_lr(self.optimizer)
        self.ent_coef = config.ent_coef
        self.clip_range = config.clip_range
        self.kl_beta = config.kl_beta
        self.model_iterations = 0
        self.value_iterations = 0
        tail = self.optimizer.bucket.tail
        self._stats = {"actor": tail[0:8], "critic": tail[8:16], "aux": tail[16:24]}
        self._scratch = _lib.scratch(self.device)
        self._gaussian = isinstance(getattr(model.actor, "actor_head", None), GaussianActorHead)
        self._zeros = {}
        self._ws = None

    def estimate_total_iterations(self):
        """ppg_learner.py:31-36."""
        buffer_size = self.config.horizon_size * self.config.parallels
        update_times = self.config.running_steps // buffer_size
        return update_times * self.config.n_epochs * self.config.n_minibatch

    def _zero_rows(self, B):
        """A persistent zero [B] vector: K4's value and return inputs in the policy phase (vf_coef = 0)."""
        if B not in self._zeros:
            self._zeros[B] = torch.zeros(B, dtype=torch.float32, device=self.device)
        return self._zeros[B]

    def _step(self, outputs, grads, segments):
        opt = self.optimizer
        opt.zero_grad()
        torch.autograd.backward(outputs, grads)
        opt.launch(max_norm=self.grad_clip_norm if self.use_grad_clip else None, segments=segments)

    # ---------------------------------------------------------------- device halves (static shapes, no host sync)
    def _device_actor(self, obs, act, adv, old_logp):
        """ppg_learner.py:50-62: the PPO-Clip surrogate minus ent_coef * entropy, through K4 / K4G with vf_coef = 0."""
        z = self._zero_rows(act.shape[0])
        st = self._stats["actor"]
        if self._gaussian:
            mu, log_std = self.model.mu_log_std(obs)
            mu, ls = mu.contiguous(), log_std.detach().contiguous()
            B, D = mu.shape
            if self._ws is None:
                self._ws = torch.empty(int(_lib.load().xb_ppo_gauss_ws_doubles(1 << 40, D)), dtype=torch.float64,
                                       device=self.device)
            dmu, dls, dz = torch.empty_like(mu), torch.empty_like(ls), torch.empty_like(z)
            _lib.call("xb_ppo_gauss_loss_fwd_bwd", _lib.ptr(mu), _lib.ptr(ls), _lib.ptr(z), _lib.ptr(act),
                      _lib.ptr(old_logp), _lib.ptr(adv), _lib.ptr(z), B, D, B, float(self.clip_range), 0.0,
                      float(self.ent_coef), 0, _lib.ptr(dmu), _lib.ptr(dls), _lib.ptr(dz), _lib.ptr(st),
                      _lib.ptr(self._scratch), _lib.ptr(self._ws), self._ws.numel())
            self._step([mu, log_std], [dmu, dls], [ACTOR])
        else:
            logits = self.model.logits(obs).contiguous()
            B, A = logits.shape
            dlogits, dz = torch.empty_like(logits), torch.empty_like(z)
            _lib.call("xb_ppo_loss_fwd_bwd", _lib.ptr(logits), _lib.ptr(z), _lib.ptr(act), _lib.ptr(old_logp),
                      _lib.ptr(adv), _lib.ptr(z), B, A, B, float(self.clip_range), 0.0, float(self.ent_coef), 0,
                      _lib.ptr(dlogits), _lib.ptr(dz), _lib.ptr(st), _lib.ptr(self._scratch))
            self._step([logits], [dlogits], [ACTOR])

    def _device_critic(self, obs, ret):
        """ppg_learner.py:98-104: MSE(critic(obs), R) through K4P with the policy and auxiliary inputs absent."""
        v = self.model.critic.values(obs).contiguous()
        dv = torch.empty_like(v)
        _lib.call("xb_ppg_aux_loss_fwd_bwd", None, None, _lib.ptr(v), None, _lib.ptr(ret), v.shape[0], 0, v.shape[0],
                  float(self.kl_beta), None, _lib.ptr(dv), None, _lib.ptr(self._stats["critic"]),
                  _lib.ptr(self._scratch))
        self._step([v], [dv], [CRITIC])

    def _device_aux(self, obs, ret, old_a, old_b=None):
        """ppg_learner.py:121-136 through K4P.  Categorical: ``old_a`` = old logits [B, A]; Gaussian: ``old_a`` = old mu
        [B, D], ``old_b`` = old log_std [D]."""
        v = self.model.critic.values(obs).contiguous()
        aux = self.model.aux_values(obs).contiguous()
        B = v.shape[0]
        dv, daux = torch.empty_like(v), torch.empty_like(aux)
        st = self._stats["aux"]
        if self._gaussian:
            mu, log_std = self.model.mu_log_std(obs)
            mu, ls = mu.contiguous(), log_std.detach().contiguous()
            dmu, dls = torch.empty_like(mu), torch.empty_like(ls)
            _lib.call("xb_ppg_aux_gauss_loss_fwd_bwd", _lib.ptr(mu), _lib.ptr(ls), _lib.ptr(old_a), _lib.ptr(old_b),
                      _lib.ptr(v), _lib.ptr(aux), _lib.ptr(ret), B, mu.shape[1], B, float(self.kl_beta),
                      _lib.ptr(dmu), _lib.ptr(dls), _lib.ptr(dv), _lib.ptr(daux), _lib.ptr(st),
                      _lib.ptr(self._scratch))
            self._step([mu, log_std, v, aux], [dmu, dls, dv, daux], [ACTOR, CRITIC, AUX])
        else:
            logits = self.model.logits(obs).contiguous()
            dlogits = torch.empty_like(logits)
            _lib.call("xb_ppg_aux_loss_fwd_bwd", _lib.ptr(logits), _lib.ptr(old_a), _lib.ptr(v), _lib.ptr(aux),
                      _lib.ptr(ret), B, logits.shape[1], B, float(self.kl_beta), _lib.ptr(dlogits), _lib.ptr(dv),
                      _lib.ptr(daux), _lib.ptr(st), _lib.ptr(self._scratch))
            self._step([logits, v, aux], [dlogits, dv, daux], [ACTOR, CRITIC, AUX])

    # ---------------------------------------------------------------- the reference's entry points
    def _obs(self, samples):
        obs = samples['obs']
        return obs if hasattr(obs, "fmt") else torch.as_tensor(obs, device=self.device)

    def _old_params(self, old_dist, old_log_std=None):
        """The old distribution's parameters as K4P takes them: Categorical logits (log-softmax normalised, which the
        kernel's normalisation leaves as they are), or (mu [B, D], log_std [D]) of a Normal whose scale every row
        shares.  ``old_log_std``: the relabel's log_std snapshot when the caller has it (the buffer passes it as
        ``aux_batch['old_dist_log_std']``); a reference-shaped caller's is recovered from row 0 of its scale."""
        if self._gaussian:
            if old_log_std is None:
                std = old_dist.std
                old_log_std = std.reshape(-1, std.shape[-1])[0].log()
            return self._f32(old_dist.mu), self._f32(old_log_std)
        return self._f32(old_dist.logits), None

    def update_actor(self, sync=True, **samples):
        """ppg_learner.py:38-88.  ``old_logp`` is ``aux_batch['old_logp']`` (the log-probabilities written at acting
        time) when present; a caller that passes only ``old_dist`` gets it from ``old_dist.log_prob(actions)``."""
        self.model_iterations += 1
        obs = self._obs(samples)
        act = self._f32(samples['actions'])
        adv = self._f32(samples['advantages'])
        aux = samples['aux_batch']
        if aux.get('old_logp') is not None:
            old_logp = self._f32(aux['old_logp'])
        else:
            old = aux['old_dist']
            a = act if self._gaussian else act.long()
            old_logp = self._f32(old.log_prob(a).detach())
        info = self.callback.on_update_start(self.iterations, method="update_model", model=self.model, obs=obs,
                                             act=act, advantages=adv, old_logp=old_logp) or {}
        self.optimizer.prepare([ACTOR])
        self._device_step(("actor", act.shape[0]), self._device_actor, obs, act, adv, old_logp)
        if self.scheduler is not None:
            self.scheduler.step()
        if not sync:
            return info
        s = self._stats["actor"].tolist()
        vals = {"actor-loss": s[0], "entropy": s[2], "learning_rate": self.optimizer.param_groups[0]['lr'],
                "clip_ratio": s[4]}
        return self._finish_info(info, vals, method="update_model", model=self.model)

    def update_critic(self, sync=True, **samples):
        """ppg_learner.py:90-112."""
        self.value_iterations += 1
        obs = self._obs(samples)
        ret = self._f32(samples['returns'])
        info = self.callback.on_update_start(self.iterations, method="update_critic", model=self.model, obs=obs,
                                             returns=ret) or {}
        self.optimizer.prepare([CRITIC])
        self._device_step(("critic", ret.shape[0]), self._device_critic, obs, ret)
        if not sync:
            return info
        vals = {"critic-loss": self._stats["critic"][2].item()}
        return self._finish_info(info, vals, method="update_critic", model=self.model)

    def update_auxiliary_critic(self, sync=True, **samples):
        """ppg_learner.py:114-148."""
        obs = self._obs(samples)
        ret = self._f32(samples['returns'])
        old = samples['aux_batch']['old_dist']
        info = self.callback.on_update_start(self.iterations, method="update_auxiliary", model=self.model, obs=obs,
                                             returns=ret, old_dist=old) or {}
        old_a, old_b = self._old_params(old, samples['aux_batch'].get('old_dist_log_std'))
        self.optimizer.prepare([ACTOR, CRITIC, AUX])
        args = (obs, ret, old_a) if old_b is None else (obs, ret, old_a, old_b)
        self._device_step(("aux", ret.shape[0]), self._device_aux, *args)
        if not sync:
            return info
        s = self._stats["aux"].tolist()
        vals = {"aux-loss": s[0], "kl-loss": s[1], "value-loss": s[2], "loss": s[3]}
        return self._finish_info(info, vals, method="update_auxiliary", model=self.model)

    def update(self, *args):
        """ppg_learner.py:150-151: PPG updates through the three phase methods."""
        return

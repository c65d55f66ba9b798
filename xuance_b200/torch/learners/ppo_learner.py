"""PPO-Clip learner - mirror of xuance/torch/learners/policy_gradient/ppo_learner.py:12-95.

``update(**samples)`` keeps the reference's signature, info keys and numerics (fp32 tolerance, tests/), but runs
as: network forward (cuDNN/cuBLAS via torch) -> K4 fused loss forward+backward (one launch producing dlogits,
dvalue and the logged statistics) -> torch backward through the network into the flat gradient bucket ->
[one NCCL all-reduce] -> K7 fused clip-norm + Adam.  No ``.item()`` until the info dict is built (one D2H of
8 floats; skipped entirely with ``sync=False`` as train_epochs does for all but the last minibatch)."""
import torch

from ... import _lib
from ..rl_models.heads import GaussianActorHead
from ..utils import FusedAdam
from .learner import Learner


class PPO_Learner(Learner):
    loss_kind = 0            # K4: 0 = PPO-Clip surrogate, 1 = plain policy gradient (A2C / PG subclasses)
    adv_key = "advantages"   # which sample field weights the log-probabilities
    info_names = ("actor_loss", "critic_loss", "entropy", "learning_rate", "predict_value", "clip_ratio")

    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        self.optimizer = FusedAdam(self.model.parameters(), self.config.learning_rate, eps=1e-5)
        self.scheduler = self._linear_lr(self.optimizer, self._lr_total_iters())
        self.vf_coef, self.ent_coef = getattr(config, "vf_coef", 0.0), config.ent_coef
        self.clip_range = getattr(config, "clip_range", 0.0)
        self._stats = self.optimizer.bucket.tail[:8]      # the logged sums travel in the gradient bucket's tail
        self._scratch = _lib.scratch(self.device)
        # a GaussianActorHead (Box action space) takes the K4G branch of _device_update
        self._gaussian = isinstance(getattr(self.model, "actor", None), GaussianActorHead)
        self._ws = None

    def _lr_total_iters(self):
        return self.total_iters

    def estimate_total_iterations(self):
        """ppo_learner.py:28-33."""
        buffer_size = self.config.horizon_size * self.config.parallels
        update_times = self.config.running_steps // buffer_size
        return update_times * self.config.n_epochs * self.config.n_minibatch

    def _gauss_ws(self, D):
        """K4G's column-partial workspace, allocated once at the size that fits any row count (D x 2048 doubles, at
        most 1 MiB): captured graphs keep the pointer they were recorded with, so it is never reallocated."""
        if self._ws is None:
            need = int(_lib.load().xb_ppo_gauss_ws_doubles(1 << 40, D))
            self._ws = torch.empty(need, dtype=torch.float64, device=self.device)
        return self._ws

    def _loss_gauss(self, obs, act, ret, adv, old_logp):
        """The Gaussian-policy branch: K4G gives (dmu, dlog_std, dvalue) and the statistics in one launch."""
        mu, log_std, v_pred = self.model.forward_raw_gauss(obs)
        mu_c, v_c = mu.contiguous(), v_pred.contiguous()
        B, D = mu_c.shape
        ls_c = log_std.detach().contiguous()
        dmu, dvalue = torch.empty_like(mu_c), torch.empty_like(v_c)
        dlog_std = torch.empty_like(ls_c)
        ws = self._gauss_ws(D)
        _lib.call("xb_ppo_gauss_loss_fwd_bwd", _lib.ptr(mu_c), _lib.ptr(ls_c), _lib.ptr(v_c), _lib.ptr(act),
                  _lib.ptr(old_logp), _lib.ptr(adv), _lib.ptr(ret), B, D, B * self.world_size, float(self.clip_range),
                  float(self.vf_coef), float(self.ent_coef), self.loss_kind, _lib.ptr(dmu), _lib.ptr(dlog_std),
                  _lib.ptr(dvalue), _lib.ptr(self._stats), _lib.ptr(self._scratch), _lib.ptr(ws), ws.numel())
        return [mu_c, v_c, log_std], [dmu, dvalue, dlog_std]

    def _device_update(self, obs, act, ret, adv, old_logp):
        """ppo_learner.py:43-65 on the device (no host synchronisation, static shapes: CUDA-graph capturable):
        loss -> backward -> [one all-reduce of gradient + statistics] -> K7."""
        loss = self._loss_gauss if self._gaussian else self._loss_categorical
        self._optimizer_step(self.optimizer, *loss(obs, act, ret, adv, old_logp))

    def _loss_categorical(self, obs, act, ret, adv, old_logp):
        B = act.shape[0]
        if hasattr(self.model, "forward_raw"):
            logits, v_pred = self.model.forward_raw(obs)
        else:
            out = self.model(obs)
            logits, v_pred = out.distributions.logits, out.values
        logits_c, v_c = logits.contiguous(), v_pred.contiguous()
        A = logits_c.shape[-1]
        dlogits = torch.empty_like(logits_c)
        dvalue = torch.empty_like(v_c)
        B_total = B * self.world_size
        _lib.call("xb_ppo_loss_fwd_bwd", _lib.ptr(logits_c), _lib.ptr(v_c), _lib.ptr(act), _lib.ptr(old_logp),
                  _lib.ptr(adv), _lib.ptr(ret), B, A, B_total, float(self.clip_range), float(self.vf_coef),
                  float(self.ent_coef), self.loss_kind, _lib.ptr(dlogits), _lib.ptr(dvalue), _lib.ptr(self._stats),
                  _lib.ptr(self._scratch))
        return [logits_c, v_c], [dlogits, dvalue]

    def host_pre_step(self):
        """Host half before the device update (step counter + 16-byte hyper-parameter upload)."""
        self.iterations += 1
        self.optimizer.prepare()

    def host_post_step(self):
        if self.scheduler is not None:
            self.scheduler.step()

    def update(self, sync=True, **samples):
        obs = samples['obs']
        if not hasattr(obs, "fmt"):  # PreparedObs passes through; arrays / tensors go to the device
            obs = torch.as_tensor(obs, device=self.device)
        act = self._f32(samples['actions'])
        ret = self._f32(samples['returns'])
        adv = self._f32(samples[self.adv_key])
        old_logp = self._f32(samples['aux_batch']['old_logp']) if self.loss_kind == 0 else None
        self.host_pre_step()
        info = self.callback.on_update_start(self.iterations, policy=self.model, obs=obs, act=act, returns=ret,
                                             advantages=adv, old_logp=old_logp) or {}
        self._device_update(obs, act, ret, adv, old_logp)
        self.host_post_step()
        if sync:
            self._finish_info(info, self._info_values(), policy=self.model)
        return info

    def materialize_info(self):
        """The logged values of the last update, with the rank suffix of a distributed run."""
        return self._with_rank(self._info_values())

    def _info_values(self):
        """The single device->host read of an update: 8 floats."""
        s = self._stats.tolist()
        lr = self.optimizer.param_groups[0]['lr']
        full = dict(zip(("actor_loss", "critic_loss", "entropy", "learning_rate", "predict_value", "clip_ratio"),
                        (s[0], s[1], s[2], lr, s[3], s[4])))
        return {name: full[name.replace("-", "_")] for name in self.info_names}


class A2C_Learner(PPO_Learner):
    """Advantage actor-critic - mirror of xuance/torch/learners/policy_gradient/a2c_learner.py:13-85:
    a_loss = -mean(adv * logp); same value / entropy terms, optimiser recipe and info keys (hyphenated, as the reference)."""
    loss_kind = 1
    info_names = ("actor-loss", "critic-loss", "entropy", "learning_rate", "predict_value")

    def _lr_total_iters(self):
        return self.config.running_steps   # a2c_learner.py:21 decays over running_steps, not over the update count


class PG_Learner(PPO_Learner):
    """Vanilla policy gradient - mirror of xuance/torch/learners/policy_gradient/pg_learner.py:12-75:
    loss = -mean(returns * logp) - ent_coef * entropy (no value term)."""
    loss_kind = 1
    adv_key = "returns"
    info_names = ("actor-loss", "entropy", "learning_rate")

    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        self.vf_coef = 0.0

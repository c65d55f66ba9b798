"""Natural policy gradient learner - mirror of xuance/torch/learners/policy_gradient/npg_learner.py:7-113.

Two optimisers as the reference's (actor and critic, lr = ``learning_rate``, eps 1e-5, each with a LinearLR over
``running_steps``), the same info keys, and the same natural gradient: for every actor parameter tensor, the
representation's included, the reference replaces the gradient g with F^-1 g where F = kappa s s^T + 1e-3 I,
s = d(sum_b log pi_b)/d(tensor) and kappa = sum_b log pi_b / horizon_size.  F is a scaled identity plus a rank-one term,
so F^-1 g has the closed form that K7N applies to the whole actor bucket in one call (include/xb200.h), instead of the
reference's dense P x P inverse per tensor.

The device half of an update: actor and critic forwards -> K4N (loss seed, score seed, critic seed, statistics, the
device sum of log pi) -> backward of the score seed, copied into the score buffer -> backward of the loss seed into the
actor bucket -> backward of the critic seed -> K7N -> the critic's and the actor's K7 clip + Adam.  No host
synchronisation: CUDA-graph capturable (``use_cuda_graph``).  Statistics are read only when ``sync`` is set."""
import numpy as np
import torch

from ... import _lib
from ..rl_models.heads import GaussianActorHead
from ..utils import FusedAdam
from .learner import Learner

FISHER_DAMPING = 1e-3       # npg_learner.py:111: F + 1e-3 * I


class NPG_Learner(Learner):
    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        if self.world_size > 1:
            raise NotImplementedError("NPG runs on one GPU: multi-GPU training is not supported")
        lr = self.config.learning_rate
        self.optimizer = {"actor": FusedAdam(self.model.actor.parameters(), lr, eps=1e-5),
                          "critic": FusedAdam(self.model.critic.parameters(), lr, eps=1e-5)}
        self.scheduler = {k: self._linear_lr(o, config.running_steps) for k, o in self.optimizer.items()}
        self.horizon_size = config.horizon_size
        self._gaussian = isinstance(getattr(model.actor, "actor_head", None), GaussianActorHead)
        bucket = self.optimizer["actor"].bucket
        self._stats = bucket.tail[:8]
        self._logp_sum = torch.zeros(1, dtype=torch.float64, device=self.device)
        self._scratch = _lib.scratch(self.device)
        self._score = torch.zeros_like(bucket.grad)
        self._table, self._nchunks = segment_table(bucket.offsets, [p.numel() for p in bucket.params], self.device)
        self._k7n_ws = torch.zeros(2 * self._nchunks, dtype=torch.float64, device=self.device)
        self._gauss_ws = None

    def _loss_seeds(self, obs, act, ret, adv):
        """K4N -> (actor outputs, their loss seeds, their score seeds, values, the critic seed)."""
        P = _lib.ptr
        v = self.model.critic.values(obs).contiguous()
        dv = torch.empty_like(v)
        B = v.shape[0]
        if self._gaussian:
            mu, log_std = self.model.mu_log_std(obs)
            mu, ls = mu.contiguous(), log_std.detach().contiguous()
            D = mu.shape[1]
            if self._gauss_ws is None:        # sized once for any row count: a captured graph keeps its pointer
                self._gauss_ws = torch.empty(int(_lib.load().xb_npg_gauss_ws_doubles(1 << 40, D)),
                                             dtype=torch.float64, device=self.device)
            dmu, smu, dls, sls = torch.empty_like(mu), torch.empty_like(mu), torch.empty_like(ls), torch.empty_like(ls)
            _lib.call("xb_npg_gauss_loss_fwd_bwd", P(mu), P(ls), P(v), P(act), P(adv), P(ret), B, D, P(dmu), P(dls),
                      P(smu), P(sls), P(dv), P(self._stats), P(self._logp_sum), P(self._scratch), P(self._gauss_ws),
                      self._gauss_ws.numel())
            return [mu, log_std], [dmu, dls], [smu, sls], v, dv
        logits = self.model.logits(obs).contiguous()
        dz, sz = torch.empty_like(logits), torch.empty_like(logits)
        _lib.call("xb_npg_loss_fwd_bwd", P(logits), P(v), P(act), P(adv), P(ret), B, logits.shape[1], P(dz), P(sz),
                  P(dv), P(self._stats), P(self._logp_sum), P(self._scratch))
        return [logits], [dz], [sz], v, dv

    def _device_natural(self, obs, act, ret, adv):
        """npg_learner.py:37-69 on the device (static shapes, no host synchronisation)."""
        actor, critic = self.optimizer["actor"], self.optimizer["critic"]
        outs, loss_seeds, score_seeds, v, dv = self._loss_seeds(obs, act, ret, adv)
        actor.zero_grad()
        torch.autograd.backward(outs, score_seeds, retain_graph=True)
        self._score.copy_(actor.bucket.grad)
        actor.zero_grad()
        torch.autograd.backward(outs, loss_seeds)
        critic.zero_grad()
        torch.autograd.backward([v], [dv])
        _lib.call("xb_npg_natural_grad", _lib.ptr(actor.bucket.grad), _lib.ptr(self._score), _lib.ptr(self._table),
                  len(actor.bucket.params), self._nchunks, _lib.ptr(self._logp_sum), float(self.horizon_size),
                  FISHER_DAMPING, _lib.ptr(self._k7n_ws), self._k7n_ws.numel())
        clip = self.grad_clip_norm if self.use_grad_clip else None
        critic.launch(max_norm=clip)
        actor.launch(max_norm=clip)

    def _obs(self, samples):
        obs = samples['obs']
        return obs if hasattr(obs, "fmt") else torch.as_tensor(obs, device=self.device)

    def update(self, sync=True, **samples):
        """npg_learner.py:26-98."""
        self.iterations += 1
        obs = self._obs(samples)
        act, ret, adv = self._f32(samples['actions']), self._f32(samples['returns']), self._f32(samples['advantages'])
        info = self.callback.on_update_start(self.iterations, model=self.model, obs=obs, act=act, returns=ret,
                                             advantages=adv) or {}
        for o in self.optimizer.values():
            o.prepare()
        self._device_step(("npg", ret.shape[0]), self._device_natural, obs, act, ret, adv)
        for k in ("critic", "actor"):
            self.scheduler[k].step()
        if not sync:
            return info
        s = self._stats.tolist()
        lr = self.optimizer["actor"].param_groups[0]['lr']
        vals = {"actor-loss": s[0], "critic-loss": s[1], "learning_rate_actor": lr,
                "learning_rate_critic": lr,      # npg_learner.py:76: the reference logs the actor's rate under both keys
                "predict_value": s[2]}
        return self._finish_info(info, vals, model=self.model)


def segment_table(offsets, lengths, device):
    """K7N's device segment table for segments at element ``offsets`` with ``lengths`` -> (table, chunk count)."""
    off = np.ascontiguousarray(offsets, np.int64)
    lens = np.ascontiguousarray(lengths, np.int64)
    table = np.zeros(3 * len(off), np.int64)
    n = int(_lib.load().xb_npg_segment_table(off.ctypes.data, lens.ctypes.data, len(off), table.ctypes.data))
    _lib.check(0 if n > 0 else n, "xb_npg_segment_table")
    return torch.from_numpy(table).to(device), n

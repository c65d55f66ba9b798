"""DQN and PER-DQN learners - mirrors of xuance/torch/learners/qlearning_family/dqn_learner.py:13-75 and
perdqn_learner.py:16-80.

update(): eval network forward (grad) + target network forward (no grad) in cuDNN/cuBLAS, then ONE K6 launch
computes the TD target, the MSE loss statistics, dLoss/dQ and the TD errors; torch backward fills the flat bucket;
[one NCCL all-reduce]; K7 clip+Adam; hard target sync every ``sync_frequency`` updates.  The importance weights of
the PER sample are ignored, as in the reference (appendix B #8)."""
import torch

from ... import _lib
from ..utils import FusedAdam
from .learner import Learner


class DQN_Learner(Learner):
    returns_td = False
    double_q = False     # DDQN_Learner: target value taken at the eval network's greedy next action

    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        params = model.eval_parameters() if hasattr(model, "eval_parameters") else model.parameters()
        self.optimizer = FusedAdam(params, self.config.learning_rate, eps=1e-5)
        self.scheduler = self._linear_lr(self.optimizer)
        self.gamma = config.gamma
        self.sync_frequency = config.sync_frequency
        self.n_actions = self.model.n_actions
        self._stats = self.optimizer.bucket.tail[:4]       # logged sums ride in the gradient all-reduce (bucket tail)
        self._scratch = _lib.scratch(self.device)
        self._graph_tensors = list(self.model.target_parameters())

    def _device_update(self, obs, nxt, act, rew, ter):
        """dqn_learner.py:38-52 on the device: no host synchronisation, static shapes (CUDA-graph capturable)."""
        evalQ = self.model(obs).values.contiguous()
        with torch.no_grad():
            targetQ = self.model.target(nxt).values.contiguous()
            selQ = self.model(nxt).values.contiguous() if self.double_q else None
        B, A = evalQ.shape
        dq = torch.empty_like(evalQ)
        td = torch.empty(B, dtype=torch.float32, device=self.device)
        _lib.call("xb_dqn_td_fwd_bwd", _lib.ptr(evalQ), _lib.ptr(targetQ), _lib.ptr(selQ), _lib.ptr(act), _lib.ptr(rew),
                  _lib.ptr(ter), B, A, B * self.world_size, float(self.gamma), _lib.ptr(dq), _lib.ptr(td),
                  _lib.ptr(self._stats), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer, [evalQ], [dq])
        return td.abs()

    def update(self, sync=True, **samples):
        self.iterations += 1
        obs = torch.as_tensor(samples['obs'], device=self.device)
        nxt = torch.as_tensor(samples['obs_next'], device=self.device)
        act, rew, ter = self._f32(samples['actions']), self._f32(samples['rewards']), self._f32(samples['terminals'])
        info = self.callback.on_update_start(self.iterations, model=self.model, obs=obs, act=act, next_obs=nxt,
                                             rew=rew, termination=ter) or {}
        self.optimizer.prepare()
        abs_td = self._device_step((tuple(obs.shape), obs.dtype), self._device_update, obs, nxt, act, rew, ter)
        if self.scheduler is not None:
            self.scheduler.step()
        if self.iterations % self.sync_frequency == 0:
            self.model.copy_target()
        if sync:
            self._finish_info(info, self._info_values(), model=self.model)
        if self.returns_td:
            return abs_td, info   # |td| stays on the device; PerOffPolicyBuffer.update_priorities takes it as is
        return info

    def _info_values(self):
        """The logged values of one update (read back from the bucket tail: the one host synchronisation)."""
        s = self._stats.tolist()
        return {"Qloss": s[0], "learning_rate": self.optimizer.param_groups[0]['lr'], "predictQ": s[1]}


class PerDQN_Learner(DQN_Learner):
    """perdqn_learner.py:80 returns (|td| [B], info)."""
    returns_td = True


class DDQN_Learner(DQN_Learner):
    """Double DQN - mirror of xuance/torch/learners/qlearning_family/ddqn_learner.py:13-80."""
    double_q = True


class DuelDQN_Learner(DQN_Learner):
    """Dueling DQN - mirror of xuance/torch/learners/qlearning_family/dueldqn_learner.py:12-80: the TD arithmetic is the DQN
    learner's (max over the target network's Q); the dueling decomposition lives in the network head."""

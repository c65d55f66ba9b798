"""C51 and QR-DQN learners - mirrors of xuance/torch/learners/qlearning_family/c51_learner.py:12-81 and
qrdqn_learner.py:12-77.

update(): the eval network's raw [B, A, N] head output (grad) and the target network's (no grad) in cuDNN/cuBLAS, then
ONE K6Z launch computes the target network's greedy action, the distributional target (C51: projected onto the
supports; QR: the quantile backup), the loss statistic and dLoss/d(raw output); torch backward fills the flat bucket;
[one NCCL all-reduce]; K7 clip+Adam; hard target sync every ``sync_frequency`` updates.  No host synchronisation before
the info dict; ``use_cuda_graph`` captures the device part per input shape, as DQN_Learner does."""
import torch

from ... import _lib
from .dqn_learner import DQN_Learner


class _DistDQN_Learner(DQN_Learner):
    def _loss(self, z, zn, act, rew, ter, grad, target_actions):
        raise NotImplementedError

    def _device_update(self, obs, nxt, act, rew, ter):
        z = self.model.forward_raw(obs).contiguous()
        zn = self.model.target_raw(nxt).contiguous()
        grad = torch.empty_like(z)
        target_actions = torch.empty(z.shape[0], dtype=torch.int64, device=z.device)
        self._loss(z, zn, act, rew, ter, grad, target_actions)
        self._optimizer_step(self.optimizer, [z], [grad])

    def _info_values(self):
        """c51_learner.py:65-74 / qrdqn_learner.py:62-71: the reference's keys, Qloss and learning_rate."""
        return {"Qloss": self._stats[0].item(), "learning_rate": self.optimizer.param_groups[0]['lr']}


class C51_Learner(_DistDQN_Learner):
    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        self.atom_num = self.model.atom_num

    def _loss(self, z, zn, act, rew, ter, grad, target_actions):
        m = self.model
        B, A, N = z.shape
        _lib.call("xb_c51_loss_fwd_bwd", _lib.ptr(z), _lib.ptr(zn), _lib.ptr(m.supports), _lib.ptr(act), _lib.ptr(rew),
                  _lib.ptr(ter), B, A, N, B * self.world_size, float(self.gamma), float(m.v_min), float(m.v_max),
                  float(m.delta_z), _lib.ptr(grad), _lib.ptr(target_actions), None, _lib.ptr(self._stats), _lib.ptr(self._scratch))


class QRDQN_Learner(_DistDQN_Learner):
    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        self.quantile_num = self.model.quantile_num

    def _loss(self, z, zn, act, rew, ter, grad, target_actions):
        B, A, N = z.shape
        _lib.call("xb_qrdqn_loss_fwd_bwd", _lib.ptr(z), _lib.ptr(zn), _lib.ptr(act), _lib.ptr(rew), _lib.ptr(ter), B, A,
                  N, B * self.world_size, float(self.gamma), _lib.ptr(grad), _lib.ptr(target_actions), _lib.ptr(self._stats),
                  _lib.ptr(self._scratch))

"""DRQN learner - mirror of xuance/torch/learners/qlearning_family/drqn_learner.py:12-80.

update(): the eval network runs K13L (or K13) over obs[:, :-1] and the target network over obs[:, 1:], both from zero
states as the reference does; ONE K6 launch over the B*L rows computes the mean-squared TD loss over every window
step (unmasked, as the reference) and dLoss/dQ (the target's own arg-max is its max, so K6's max target is the
reference's); the backward runs through K13L into the flat bucket; K7 clip + Adam (eps 1e-5); LinearLR every update;
hard target sync every ``sync_frequency`` updates.  The device half is keyed on the window length for CUDA graphs."""
import torch

from ... import _lib
from .dqn_learner import DQN_Learner


class DRQN_Learner(DQN_Learner):
    def __init__(self, config, model, callback):
        super().__init__(config, model, callback)
        if self.world_size > 1:
            raise NotImplementedError("DRQN_Learner: distributed training is not supported (one rank)")

    def _device_update(self, obs, act, rew, ter):
        _, out = self.model(obs[:, :-1])
        evalQ = out.values.contiguous()
        with torch.no_grad():
            _, tout = self.model.target(obs[:, 1:])
            targetQ = tout.values.contiguous()
        B, L, A = evalQ.shape
        dq = torch.empty_like(evalQ)
        td = torch.empty(B * L, dtype=torch.float32, device=self.device)
        _lib.call("xb_dqn_td_fwd_bwd", _lib.ptr(evalQ), _lib.ptr(targetQ), None, _lib.ptr(act), _lib.ptr(rew),
                  _lib.ptr(ter), B * L, A, B * L, float(self.gamma), _lib.ptr(dq), _lib.ptr(td),
                  _lib.ptr(self._stats), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer, [evalQ], [dq])

    def update(self, sync=True, **samples):
        self.iterations += 1
        obs = self._f32(samples['obs'])
        act, rew, ter = self._f32(samples['actions']), self._f32(samples['rewards']), self._f32(samples['terminals'])
        info = self.callback.on_update_start(self.iterations, model=self.model, obs=obs, act=act, rew=rew,
                                             termination=ter, batch_size=samples.get('batch_size')) or {}
        self.optimizer.prepare()
        self._device_step(tuple(obs.shape), self._device_update, obs, act, rew, ter)
        if self.scheduler is not None:
            self.scheduler.step()
        if self.iterations % self.sync_frequency == 0:
            self.model.copy_target()
        if sync:
            self._finish_info(info, self._info_values(), model=self.model)
        return info

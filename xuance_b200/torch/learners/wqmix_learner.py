"""Weighted QMIX learner (OW-QMIX / CW-QMIX) - mirror of xuance/torch/learners/multi_agent_rl/wqmix_learner.py:15-227
for one parameter-sharing group with GRU agents (use_rnn=True).

update(sample): agent and central agent networks over the padded episodes (cuDNN GRU) for eval (grad) and target (no
grad) -> K9W select (the taken eval values, the central values at the greedy actions, the target central values at the
next actions, greedy indices, CW agreement flags, sum(filled)) -> QMIX mixer (hypernet GEMMs + K9 mix) and feed-forward
mixers (cuBLAS) -> K9W weighted loss (dQtot, dQff + statistics) -> torch backward through both mixers, the selection
(K9W select backward) and both agent networks -> [one NCCL all-reduce] -> K7.

The weighting follows ``config.agent``: "OWQMIX" (w = 1 where td < 0) or "CWQMIX" (w = 1 where every agent's taken action
is its greedy one, or where y > Q_ff), alpha elsewhere.

``config.qmix_rnn_detach_q_eval`` (default False): the reference slices q_eval and q_eval_centralized inside
torch.no_grad() (wqmix_learner.py:46-66), so with use_rnn neither the agent networks nor the central agent networks
receive any gradient - only the two mixers train.  True reproduces that bit for bit; False (default) runs the evidently
intended computation.  DESIGN.md "Reference quirks"."""
import torch

from ... import _lib
from ..utils import allreduce_sum_
from .qmix_learner import QMIX_Learner

_MODES = {"OWQMIX": 0, "CWQMIX": 1}     # XB_WQMIX_OW / XB_WQMIX_CW


class _WeightedSelectFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q_all, q_cent, q_cent_tgt, q_tgt, actions, agent_mask, filled, double_q, filled_sum, scratch,
                avail=None):
        B, n, T1, A = q_all.shape
        T = T1 - 1
        dev = q_all.device
        q_eval = torch.empty((B * T, n), dtype=torch.float32, device=dev)
        q_cent_taken = torch.empty((B * T, n), dtype=torch.float32, device=dev)
        q_next_cent = torch.empty((B * T, n), dtype=torch.float32, device=dev)
        greedy = torch.empty((B, n, T), dtype=torch.int32, device=dev)
        agree = torch.empty(B * T, dtype=torch.uint8, device=dev)
        if avail is not None:
            assert avail.dtype == torch.uint8 and avail.is_contiguous() and tuple(avail.shape[:3]) == (B, n, T1)
        _lib.call("xb_wqmix_select_fwd", _lib.ptr(q_all), _lib.ptr(q_cent), _lib.ptr(q_cent_tgt), _lib.ptr(q_tgt),
                  _lib.ptr(actions), _lib.ptr(agent_mask), _lib.ptr(filled), _lib.ptr(avail),
                  avail.shape[3] if avail is not None else 0, B, n, T, A, 1 if double_q else 0, _lib.ptr(q_eval),
                  _lib.ptr(q_cent_taken), _lib.ptr(q_next_cent), _lib.ptr(greedy), _lib.ptr(agree),
                  _lib.ptr(filled_sum), _lib.ptr(scratch))
        ctx.save_for_backward(actions, greedy, agent_mask, filled)
        ctx.dims = (B, n, T, A)
        ctx.mark_non_differentiable(q_next_cent, greedy, agree)
        return q_eval, q_cent_taken, q_next_cent, greedy, agree

    @staticmethod
    def backward(ctx, d_eval, d_cent, *_):
        actions, greedy, agent_mask, filled = ctx.saved_tensors
        B, n, T, A = ctx.dims
        d_eval = d_eval.contiguous() if ctx.needs_input_grad[0] and d_eval is not None else None
        d_cent = d_cent.contiguous() if ctx.needs_input_grad[1] and d_cent is not None else None
        zeros = lambda: torch.zeros((B, n, T + 1, A), dtype=torch.float32, device=greedy.device)
        dq_all = zeros() if d_eval is not None else None
        dq_cent = zeros() if d_cent is not None else None
        if d_eval is not None or d_cent is not None:
            _lib.call("xb_wqmix_select_bwd", _lib.ptr(d_eval), _lib.ptr(d_cent), _lib.ptr(actions), _lib.ptr(greedy),
                      _lib.ptr(agent_mask), _lib.ptr(filled), B, n, T, A, _lib.ptr(dq_all), _lib.ptr(dq_cent))
        return dq_all, dq_cent, None, None, None, None, None, None, None, None, None


class WQMIX_Learner(QMIX_Learner):
    """wqmix_learner.py:15-227.  Shares the episode plumbing, the optimiser set-up (one FusedAdam over the model's
    ``parameters_model``: agent networks, QMIX mixer, central agent networks, feed-forward mixer) and the graphed device
    step with QMIX_Learner."""

    def __init__(self, config, agent_grouping, model, callback):
        agent = getattr(config, "agent", None)
        if agent not in _MODES:
            raise AttributeError(f"The agent named is {agent} is currently not supported.")
        if not getattr(config, "use_rnn", False):
            raise NotImplementedError("hot-path scope: Weighted QMIX with use_rnn=True (the sc2 configurations)")
        super().__init__(config, agent_grouping, model, callback)
        self.mode = _MODES[agent]
        self.alpha = config.alpha
        self._stats = self.optimizer.bucket.tail[:4]       # logged sums ride in the gradient all-reduce (bucket tail)

    def _device_update(self, obs, actions, rewards, terminals, agent_mask, filled, state, avail=None):
        """wqmix_learner.py:131-209 on the device (no host synchronisation, static shapes: CUDA-graph capturable)."""
        B, n, T1 = obs.shape[0], obs.shape[1], obs.shape[2]
        T = T1 - 1
        packed = obs.flatten(0, 1)                                          # [B*n, T+1, obs]
        shape = (B, n, T + 1, -1)
        q_all = self.model.q_values(packed).reshape(shape).contiguous()
        q_cent = self.model.q_centralized(packed).reshape(shape).contiguous()
        with torch.no_grad():
            q_cent_tgt = self.model.q_centralized(packed, target=True).reshape(shape).contiguous()
            q_tgt = None if self.double_q else self.model.q_values(packed, target=True).reshape(shape).contiguous()
        if self.detach_q_eval:
            q_all, q_cent = q_all.detach(), q_cent.detach()
        q_eval_taken, q_cent_taken, q_next_cent, _, agree = _WeightedSelectFunction.apply(
            q_all, q_cent, q_cent_tgt, q_tgt, actions, agent_mask, filled, self.double_q, self._filled_sum,
            self._scratch, avail)
        if self.world_size > 1:
            allreduce_sum_(self._filled_sum)                                # global sum(filled) for the loss
        q_tot = self.model.Q_tot(q_eval_taken, state[:, :-1]).reshape(-1).contiguous()
        q_ff = self.model.q_feedforward(q_cent_taken, state[:, :-1]).reshape(-1).contiguous()
        with torch.no_grad():
            q_ff_next = self.model.target_q_feedforward(q_next_cent, state[:, 1:]).reshape(-1).contiguous()
        dq_tot, dq_ff = torch.empty_like(q_tot), torch.empty_like(q_ff)
        _lib.call("xb_wqmix_loss_fwd_bwd", _lib.ptr(q_tot), _lib.ptr(q_ff), _lib.ptr(q_ff_next), _lib.ptr(rewards),
                  _lib.ptr(terminals), _lib.ptr(filled), _lib.ptr(agree), _lib.ptr(self._filled_sum), B, n, T,
                  self.mode, float(self.alpha), float(self.gamma), B * T * self.world_size, _lib.ptr(dq_tot),
                  _lib.ptr(dq_ff), _lib.ptr(self._stats), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer, [q_tot, q_ff], [dq_tot, dq_ff])
        return None

    def _info(self):
        s = self._stats.tolist()
        return {"learning_rate": self.optimizer.param_groups[0]['lr'], "loss_Qmix": s[0], "loss_central": s[1],
                "loss": s[2], "predictQ": s[3]}

"""IQL learner - mirror of xuance/torch/learners/multi_agent_rl/iql_learner.py:13-142 for one parameter-sharing group of
GRU agents (use_rnn=True).

update(sample): eval agent network over the padded episodes (K13 GRU + Q head) -> target agent network (no grad) ->
``xb_iql_prepare`` (the global sum(agent_mask * filled)) -> [all-reduce of that double when sharded] -> K9I
``xb_iql_td_fwd_bwd`` (greedy next actions, masked target values, the per-agent TD loss and the whole dq_all in one
launch) -> one torch backward into the flat bucket -> [one NCCL all-reduce] -> K7.  No host synchronisation before the
info dict, so the device half is CUDA-graph capturable.

The reference slices q_eval to its first T steps inside torch.no_grad() (iql_learner.py:49-60), so with use_rnn=True its
loss has no graph and ``loss.backward()`` raises; with action masks it also slices the agent axis of the next-step masks
(:78).  This learner trains the evidently intended computation: q_eval keeps its graph, and the masks of steps 1..T are
applied.  DESIGN.md section 4."""
import torch

from ... import _lib
from ..utils import FusedAdam, allreduce_sum_
from .qmix_learner import QMIX_Learner


class IQL_Learner(QMIX_Learner):
    """iql_learner.py:13-142.  Shares the episode plumbing and the graphed device step with QMIX_Learner; one FusedAdam
    (eps 1e-5, LinearLR) over the group's agent network (IndependentMixer has no parameters), clipped when
    ``use_grad_clip``; logged values are keyed by group."""

    def __init__(self, config, agent_grouping, model, callback):
        if not getattr(config, "use_rnn", False):
            raise NotImplementedError("hot-path scope: IQL with use_rnn=True (the sc2 configurations)")
        if getattr(config, "qmix_rnn_detach_q_eval", False):
            raise NotImplementedError("IQL: qmix_rnn_detach_q_eval=True would detach the only trained term (there is "
                                      "no mixer), so nothing would train")
        super().__init__(config, agent_grouping, model, callback)
        self.group = agent_grouping.group_keys[0]
        self._msum = torch.zeros(1, dtype=torch.float64, device=self.device)
        self._graph_tensors = [self._msum]

    def _build_optimizer(self):
        # the K13 GRU reads its weights wherever they sit: no cuDNN front group
        return FusedAdam(self.model.parameters_model, lr=self.learning_rate, eps=1e-5,
                         weight_decay=getattr(self.config, "weight_decay", 0.0))

    def _uses_global_state(self):
        """IQL's replay keeps no global state."""
        return False

    def _device_update(self, obs, actions, rewards, terminals, agent_mask, filled, state, avail=None):
        """iql_learner.py:37-129 on the device (no host synchronisation, static shapes: CUDA-graph capturable)."""
        B, n, T1 = obs.shape[0], obs.shape[1], obs.shape[2]
        T = T1 - 1
        packed = obs.flatten(0, 1)                                          # [B*n, T+1, obs]
        q_all = self.model.q_values(packed).reshape(B, n, T1, -1).contiguous()
        with torch.no_grad():
            q_tgt = self.model.q_values(packed, target=True).reshape(B, n, T1, -1).contiguous()
        A = q_all.shape[-1]
        _lib.call("xb_iql_prepare", _lib.ptr(agent_mask), _lib.ptr(filled), B, n, T, _lib.ptr(self._msum),
                  _lib.ptr(self._scratch))
        if self.world_size > 1:
            allreduce_sum_(self._msum)                                      # global sum(agent_mask * filled)
        dq_all = torch.empty_like(q_all)
        _lib.call("xb_iql_td_fwd_bwd", _lib.ptr(q_all.detach()), _lib.ptr(q_tgt), _lib.ptr(actions),
                  _lib.ptr(rewards), _lib.ptr(terminals), _lib.ptr(agent_mask), _lib.ptr(filled), _lib.ptr(avail),
                  avail.shape[3] if avail is not None else 0, _lib.ptr(self._msum), B, n, T, A,
                  int(bool(self.double_q)), float(self.gamma), B * n * T * self.world_size, _lib.ptr(dq_all),
                  _lib.ptr(self._stats), _lib.ptr(self._scratch), None, None, None)
        self._optimizer_step(self.optimizer, [q_all], [dq_all])
        return None

    def _info(self):
        s = self._stats.tolist()
        g = self.group
        return {f"{g}/learning_rate": self.optimizer.param_groups[0]['lr'], f"{g}/loss_Q": s[0], f"{g}/predictQ": s[1]}

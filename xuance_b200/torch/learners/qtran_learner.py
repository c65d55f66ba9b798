"""QTRAN learner (QTRAN_base and QTRAN_alt) - mirror of xuance/torch/learners/multi_agent_rl/qtran_learner.py:199-371
(update_rnn) for one parameter-sharing group with GRU agents (use_rnn=True).

update(sample): eval and target agent networks over the padded episodes (K13 GRU + Q head) -> K9Q select (greedy actions
at every step, next actions, sum(filled)) -> three K9Q encodings: taken actions (trained), greedy actions and, with the
target network, next actions (no grad) -> Q_jt on each and V_jt (cuBLAS) -> K9Q loss (TD, opt, nopt: dQ_jt, dV and the
scatter into the agents' Q heads) -> one torch backward -> [one NCCL all-reduce] -> K7.

As the reference does: the target joint network reads the target GRU outputs of steps 0..T-1 (with the states and next
actions of steps 1..T), ``double_q`` changes only the next actions, the nopt minimum runs over unavailable actions too,
dead agents' one-hot actions still enter the encoding, alt's n per-agent terms share one V, and no gradient clipping
runs whatever ``use_grad_clip`` says.  DESIGN.md "Reference quirks"."""
import torch

from ... import _lib
from ..utils import FusedAdam, allreduce_sum_
from ..rl_models.qtran import ALT
from .qmix_learner import QMIX_Learner

_AGENTS = ("QTRAN_base", "QTRAN_alt")


class QTRAN_Learner(QMIX_Learner):
    """qtran_learner.py:17-371.  Shares the episode plumbing and the graphed device step with QMIX_Learner; one FusedAdam
    (eps 1e-5, LinearLR) over ``parameters_model``: qtran_net, the (parameter-free) VDN mixer and the agent networks."""

    def __init__(self, config, agent_grouping, model, callback):
        agent = getattr(config, "agent", None)
        if agent not in _AGENTS:
            raise ValueError("Mixer {} not recognised.".format(agent))
        if not getattr(config, "use_rnn", False):
            raise NotImplementedError("hot-path scope: QTRAN with use_rnn=True (the sc2 configurations)")
        self.lambda_opt, self.lambda_nopt = config.lambda_opt, config.lambda_nopt
        super().__init__(config, agent_grouping, model, callback)
        self.use_grad_clip = False          # update_rnn never clips (qtran_learner.py:351-353)
        self._stats = self.optimizer.bucket.tail[:5]

    def _build_optimizer(self):
        # the K13 GRU reads its weights wherever they sit: no cuDNN front group
        return FusedAdam(self.model.parameters_model, lr=self.learning_rate, eps=1e-5,
                         weight_decay=getattr(self.config, "weight_decay", 0.0))

    def _device_update(self, obs, actions, rewards, terminals, agent_mask, filled, state, avail=None):
        """qtran_learner.py:199-353 on the device (no host synchronisation, static shapes: CUDA-graph capturable)."""
        m = self.model
        net, tnet = m.qtran_net, m.target_qtran_net
        B, n, T1 = obs.shape[0], obs.shape[1], obs.shape[2]
        T = T1 - 1
        dev = obs.device
        packed = obs.flatten(0, 1)                                          # [B*n, T+1, obs]
        q_all, h = m.q_and_hidden(packed)
        A, H = q_all.shape[-1], h.shape[-1]
        q_all, h = q_all.reshape(B, n, T1, A).contiguous(), h.reshape(B, n, T1, H).contiguous()
        with torch.no_grad():
            q_tgt, h_tgt = m.q_and_hidden(packed, target=True)
            q_tgt, h_tgt = q_tgt.reshape(B, n, T1, A).contiguous(), h_tgt.reshape(B, n, T1, H).contiguous()
        greedy = torch.empty((B, n, T1), dtype=torch.int32, device=dev)
        nxt = torch.empty((B, n, T), dtype=torch.int32, device=dev)
        _lib.call("xb_qtran_select", _lib.ptr(q_all.detach()), _lib.ptr(q_tgt), _lib.ptr(avail),
                  avail.shape[3] if avail is not None else 0, _lib.ptr(filled), B, n, T, A, int(bool(self.double_q)),
                  _lib.ptr(greedy), _lib.ptr(nxt), _lib.ptr(self._filled_sum), _lib.ptr(self._scratch))
        if self.world_size > 1:
            allreduce_sum_(self._filled_sum)                                # global sum(filled) for the loss
        q_joint = net.Q_jt(net.encode(state, 0, h, agent_mask, actions))
        v = net.V_jt(state[:, :-1].reshape(B * T, -1)).reshape(-1)
        with torch.no_grad():
            q_joint_greedy = net.Q_jt(net.encode(state, 0, h.detach(), agent_mask, greedy))
            q_joint_next = tnet.Q_jt(tnet.encode(state, 1, h_tgt, agent_mask, nxt))   # h of steps 0..T-1 (:243)
        dq_joint = torch.empty_like(q_joint)
        dv = torch.empty_like(v)
        dq_all = torch.zeros_like(q_all)
        _lib.call("xb_qtran_loss_fwd_bwd", net.mode, _lib.ptr(q_all.detach()), _lib.ptr(actions), _lib.ptr(greedy),
                  _lib.ptr(nxt), _lib.ptr(agent_mask), _lib.ptr(filled), _lib.ptr(rewards), _lib.ptr(terminals),
                  _lib.ptr(q_joint.detach()), _lib.ptr(q_joint_greedy), _lib.ptr(q_joint_next), _lib.ptr(v.detach()),
                  _lib.ptr(self._filled_sum), B, n, T, A, float(self.gamma), float(self.lambda_opt),
                  float(self.lambda_nopt), B * T * self.world_size, _lib.ptr(dq_joint), _lib.ptr(dv), _lib.ptr(dq_all),
                  _lib.ptr(self._stats), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer, [q_joint, v, q_all], [dq_joint, dv, dq_all])
        return None

    def _info(self):
        s = self._stats.tolist()
        return {"learning_rate": self.optimizer.param_groups[0]['lr'], "loss_td": s[0], "loss_opt": s[1],
                "loss_nopt": s[2], "loss": s[3], "Q_joint": s[4]}

"""DCG learner (DCG and DCG_S) - mirror of xuance/torch/learners/multi_agent_rl/dcg_learner.py:19-219 for one
parameter-sharing group with GRU agents (use_rnn=True).

update(sample): eval and target representations over the padded episodes (K13 GRU) -> eval and target utility and payoff
heads over all T+1 steps (cuBLAS) -> K9C greedy on the detached eval heads at steps 1..T (the next actions) -> K9C Q
(Q_eval from the eval heads at 0..T-1 with the taken actions, Q_next from the target heads at 1..T with the greedy ones,
sum(filled)) -> [DCG_S: V(s), V(s') from the online state-value head] -> K9C TD (dq, dV + statistics) -> K9C scatter
of dq into the head outputs -> torch backward through the heads and the GRU -> [one NCCL all-reduce] -> K7.

As the reference does: ``double_q`` is read by nothing (the next actions are always the eval heads' greedy ones,
evaluated by the target heads), ``agent_mask`` is ignored (dead agents' utilities count), V(s') of DCG_S comes from the
online ``bias`` head, and ``n_msg_iterations: 0`` or a graph without edges drops the payoffs - and, for DCG_S, V(s) -
from Q.  DESIGN.md "Reference quirks"."""
import torch

from ... import _lib
from ..utils import FusedAdam, allreduce_sum_
from ..rl_models.dcg import dcg_greedy
from .qmix_learner import QMIX_Learner

_AGENTS = ("DCG", "DCG_S")


class _QFunction(torch.autograd.Function):
    """(f_eval, pay_eval) -> float64 q_eval [B*T] (with q_next and sum(filled) as non-differentiable side outputs)."""

    @staticmethod
    def forward(ctx, f_eval, pay_eval, f_tgt, pay_tgt, actions, greedy, filled, graph, use_payoff, filled_sum,
                scratch):
        B, n, T1, A = f_eval.shape
        T = T1 - 1
        dev = f_eval.device
        q_eval = torch.empty(B * T, dtype=torch.float64, device=dev)
        q_next = torch.empty(B * T, dtype=torch.float64, device=dev)
        ld = lambda p: p[0].numel() if p is not None else 0
        _lib.call("xb_dcg_q_fwd", _lib.ptr(f_eval), _lib.ptr(pay_eval), ld(pay_eval), _lib.ptr(f_tgt),
                  _lib.ptr(pay_tgt), ld(pay_tgt), _lib.ptr(actions), _lib.ptr(greedy), _lib.ptr(filled),
                  _lib.ptr(graph.edges_from), _lib.ptr(graph.edges_to), B, n, T, A, graph.n_edges, int(use_payoff),
                  _lib.ptr(q_eval), _lib.ptr(q_next), _lib.ptr(filled_sum), _lib.ptr(scratch))
        ctx.save_for_backward(actions)
        ctx.graph, ctx.dims, ctx.use_payoff, ctx.has_pay = graph, (B, n, T, A), use_payoff, pay_eval is not None
        ctx.mark_non_differentiable(q_next)
        return q_eval, q_next

    @staticmethod
    def backward(ctx, dq, _dq_next):
        actions, = ctx.saved_tensors
        B, n, T, A = ctx.dims
        graph = ctx.graph
        E = graph.n_edges
        dev = actions.device
        df = torch.zeros((B, n, T + 1, A), dtype=torch.float32, device=dev)
        dp = torch.zeros((2, B, E, T + 1, A * A), dtype=torch.float32, device=dev) if ctx.has_pay else None
        _lib.call("xb_dcg_q_bwd", _lib.ptr(dq.contiguous()), _lib.ptr(actions), _lib.ptr(graph.edges_from),
                  _lib.ptr(graph.edges_to), B, n, T, A, E, int(ctx.use_payoff), _lib.ptr(df), _lib.ptr(dp),
                  dp[0].numel() if dp is not None else 0)
        return df, dp, None, None, None, None, None, None, None, None, None


class DCG_Learner(QMIX_Learner):
    """dcg_learner.py:19-219.  Shares the episode plumbing and the graphed device step with QMIX_Learner; one FusedAdam
    (eps 1e-5, LinearLR) over ``parameters_model``: representation, utility, payoffs and, for DCG_S, the bias head."""

    def __init__(self, config, agent_grouping, model, callback):
        agent = getattr(config, "agent", None)
        if agent not in _AGENTS:
            raise AttributeError(f"The agent named is {agent} is currently not supported.")
        if not getattr(config, "use_rnn", False):
            raise NotImplementedError("hot-path scope: DCG with use_rnn=True (the sc2 configurations)")
        self.dcg_s = agent == "DCG_S"
        super().__init__(config, agent_grouping, model, callback)

    def _build_optimizer(self):
        # the K13 GRU reads its weights wherever they sit: no cuDNN front group
        return FusedAdam(self.model.parameters_model, lr=self.learning_rate, eps=1e-5,
                         weight_decay=getattr(self.config, "weight_decay", 0.0))

    def _uses_global_state(self):
        """Only DCG_S reads the global state (V(s)); DCG's replay keeps none."""
        return self.dcg_s

    def _device_update(self, obs, actions, rewards, terminals, agent_mask, filled, state, avail=None):
        """dcg_learner.py:106-215 on the device (no host synchronisation, static shapes: CUDA-graph capturable)."""
        m = self.model
        B, n, T1 = obs.shape[0], obs.shape[1], obs.shape[2]
        T = T1 - 1
        packed = obs.flatten(0, 1)                                          # [B*n, T+1, obs]
        h = m.hidden_states(packed).reshape(B, n, T1, -1)
        f_eval, pay_eval = m.heads(h)
        with torch.no_grad():
            h_tgt = m.hidden_states(packed, target=True).reshape(B, n, T1, -1)
            f_tgt, pay_tgt = m.heads(h_tgt, target=True)
            greedy = dcg_greedy(f_eval.detach(), None if pay_eval is None else pay_eval.detach(), m.graph,
                                m.n_msg_iterations, m.msg_normalized, T, 1, avail)
        q_eval, q_next = _QFunction.apply(f_eval, pay_eval, f_tgt, pay_tgt, actions, greedy, filled, m.graph,
                                          m.use_payoff, self._filled_sum, self._scratch)
        if self.world_size > 1:
            allreduce_sum_(self._filled_sum)                                # global sum(filled) for the loss
        v = v_next = dv = None
        # q_dcg returns before adding V(s) when it drops the payoffs (dcg_learner.py:95-103): then V is not in Q or Q'
        # and the state-value head gets no gradient
        use_v = self.dcg_s and m.use_payoff
        if use_v:
            S = state.shape[-1]
            v = m.state_value(state[:, :-1].reshape(B * T, S)).contiguous()
            with torch.no_grad():
                v_next = m.state_value(state[:, 1:].reshape(B * T, S)).contiguous()   # the ONLINE head, as the reference
            dv = torch.empty_like(v)
        dq = torch.empty_like(q_eval)
        _lib.call("xb_dcg_td_fwd_bwd", _lib.ptr(q_eval), _lib.ptr(q_next), _lib.ptr(v), _lib.ptr(v_next),
                  _lib.ptr(rewards), _lib.ptr(terminals), _lib.ptr(filled), _lib.ptr(self._filled_sum), B, n, T,
                  float(self.gamma), B * T * self.world_size, _lib.ptr(dq), _lib.ptr(dv), _lib.ptr(self._stats),
                  _lib.ptr(self._scratch))
        outs, grads = [q_eval], [dq]
        if use_v:
            outs.append(v)
            grads.append(dv)
        self._optimizer_step(self.optimizer, outs, grads)
        return None

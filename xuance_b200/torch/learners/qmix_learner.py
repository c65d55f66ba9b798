"""QMIX learner - mirror of xuance/torch/learners/multi_agent_rl/qmix_learner.py:12-112 (+ its parents
iql_learner.py:37-83 and base/marl_learner.py:18-76, 319-408) for one parameter-sharing group with GRU agents.

update(sample): agent network over the padded episodes (cuDNN GRU) for eval (grad) and target (no grad) ->
K9 select (gathers, double-Q argmax, masks, agent-minor transpose, sum(filled)) -> eval mixer (hypernet GEMMs +
fused K9 mix) and target mixer -> K9 masked TD loss (dQtot + statistics) -> torch backward through the mixer
(K9 mix backward), the selection (K9 select backward) and the agent networks -> [one NCCL all-reduce] -> K7.

``config.qmix_rnn_detach_q_eval`` (default False): the reference at 4f0b05b slices q_eval inside torch.no_grad()
(iql_learner.py:57-59), so its agent networks receive NO gradient when use_rnn=True - only the mixer trains
(pinned in tests/test_oracle_vs_reference.py).  True reproduces that bit for bit; False (default) runs the
evidently intended computation.  DESIGN.md "Reference quirks"."""
import torch

from ... import _lib
from ..utils import FusedAdam, allreduce_sum_
from ..utils.flat_bucket import cudnn_rnn_front
from .learner import Learner


class _SelectFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q_all, q_tgt, actions, agent_mask, filled, double_q, filled_sum, scratch, avail=None):
        B, n, T1, A = q_all.shape
        T = T1 - 1
        q_eval = torch.empty((B * T, n), dtype=torch.float32, device=q_all.device)
        q_next = torch.empty((B * T, n), dtype=torch.float32, device=q_all.device)
        if avail is not None:
            assert avail.dtype == torch.uint8 and avail.is_contiguous() and tuple(avail.shape[:3]) == (B, n, T1)
        _lib.call("xb_qmix_select_fwd", _lib.ptr(q_all), _lib.ptr(q_tgt), _lib.ptr(actions), _lib.ptr(agent_mask),
                  _lib.ptr(filled), _lib.ptr(avail), avail.shape[3] if avail is not None else 0, B, n, T, A,
                  1 if double_q else 0, _lib.ptr(q_eval), _lib.ptr(q_next), _lib.ptr(filled_sum), _lib.ptr(scratch))
        ctx.save_for_backward(actions, agent_mask, filled)
        ctx.dims = (B, n, T, A)
        ctx.mark_non_differentiable(q_next)
        return q_eval, q_next

    @staticmethod
    def backward(ctx, d_eval, _d_next):
        actions, agent_mask, filled = ctx.saved_tensors
        B, n, T, A = ctx.dims
        dq_all = torch.zeros((B, n, T + 1, A), dtype=torch.float32, device=d_eval.device)
        _lib.call("xb_qmix_select_bwd", _lib.ptr(d_eval.contiguous()), _lib.ptr(actions), _lib.ptr(agent_mask),
                  _lib.ptr(filled), B, n, T, A, _lib.ptr(dq_all))
        return dq_all, None, None, None, None, None, None, None, None


class QMIX_Learner(Learner):
    rank_suffix = False

    def __init__(self, config, agent_grouping, model, callback):
        super().__init__(config, model, callback)
        self.use_parameter_sharing = getattr(config, "use_parameter_sharing", True)
        self.agent_grouping = agent_grouping
        self.agent_keys = agent_grouping.agent_keys
        self.n_agents = len(self.agent_keys)
        self.sync_frequency = config.sync_frequency
        self.double_q = getattr(config, "double_q", True)
        self.detach_q_eval = getattr(config, "qmix_rnn_detach_q_eval", False)
        self.use_actions_mask = getattr(config, "use_actions_mask", False)
        # LearnerMAS.build_optimizer (marl_learner.py:64-76): one Adam(eps=1e-5) + LinearLR over the trainable set
        self.optimizer = self._build_optimizer()
        self.scheduler = self._linear_lr(self.optimizer)
        dev = self.device
        self._filled_sum = torch.zeros(1, dtype=torch.float32, device=dev)
        self._stats = self.optimizer.bucket.tail[:2]       # logged sums ride in the gradient all-reduce (bucket tail)
        self._scratch = _lib.scratch(dev)
        self._graph_tensors = [self._filled_sum]

    def _build_optimizer(self):
        """One FusedAdam over ``parameters_model``, the cuDNN GRU weights first in the bucket (cudnn_rnn_front)."""
        return FusedAdam(self.model.parameters_model, lr=self.learning_rate, eps=1e-5,
                         weight_decay=getattr(self.config, "weight_decay", 0.0),
                         front=cudnn_rnn_front(self.model.individual_q_networks))

    def estimate_total_iterations(self):
        """marl_learner.py:37-47."""
        start_training = getattr(self.config, "start_training", 0)
        training_frequency = getattr(self.config, "training_frequency", 1)
        n_epochs = getattr(self.config, "n_epochs", 1)
        if self.use_rnn:
            total = (self.config.running_steps - start_training) // (self.episode_length * self.config.parallels)
        else:
            total = (self.config.running_steps - start_training) // (training_frequency * self.config.parallels)
        return total * n_epochs

    def _stacked(self, sample):
        """[B, n, ...] device tensors from a sample dict (uses the buffer's pre-stacked tensors when present)."""
        f32 = self._f32
        u8 = lambda x: torch.as_tensor(x, device=self.device).to(torch.uint8).contiguous()
        if '_stacked' in sample:
            st = sample['_stacked']
            out = {k: f32(st[k]) for k in ('obs', 'actions', 'rewards', 'terminals', 'agent_mask', 'filled')}
            out['state'] = f32(st['state']) if self._uses_global_state() else None
            out['avail'] = u8(st['avail_actions']) if self.use_actions_mask else None
            return out
        stack = lambda d: torch.stack([torch.as_tensor(d[a], device=self.device) for a in self.agent_keys], dim=1)
        out = {k: f32(stack(sample[k])) for k in ('obs', 'actions', 'rewards', 'terminals', 'agent_mask')}
        out['filled'] = f32(sample['filled'])
        out['state'] = f32(sample['state']) if self._uses_global_state() else None
        out['avail'] = u8(stack(sample['avail_actions'])) if self.use_actions_mask else None
        return out

    def _uses_global_state(self):
        """Whether the update reads the global state (the mixers do; a learner whose replay keeps none says False)."""
        return True

    def _device_update(self, obs, actions, rewards, terminals, agent_mask, filled, state, avail=None):
        """qmix_learner.py:24-95 on the device (no host synchronisation, static shapes: CUDA-graph capturable)."""
        B, n, T1 = obs.shape[0], obs.shape[1], obs.shape[2]
        T = T1 - 1
        packed = obs.flatten(0, 1)                                          # [B*n, T+1, obs]
        q_all = self.model.q_values(packed).reshape(B, n, T + 1, -1).contiguous()
        with torch.no_grad():
            q_tgt = self.model.q_values(packed, target=True).reshape(B, n, T + 1, -1).contiguous()
        q_in = q_all.detach() if self.detach_q_eval else q_all
        q_eval_taken, q_next_taken = _SelectFunction.apply(q_in, q_tgt, actions, agent_mask, filled, self.double_q,
                                                           self._filled_sum, self._scratch, avail)
        if self.world_size > 1:
            allreduce_sum_(self._filled_sum)                                # global sum(filled) for the loss
        q_tot_eval = self.model.Q_tot(q_eval_taken, state[:, :-1]).reshape(-1).contiguous()
        with torch.no_grad():
            q_tot_next = self.model.Qtarget_tot(q_next_taken, state[:, 1:]).reshape(-1).contiguous()
        dq_tot = torch.empty_like(q_tot_eval)
        _lib.call("xb_qmix_td", _lib.ptr(q_tot_eval), _lib.ptr(q_tot_next), _lib.ptr(rewards), _lib.ptr(terminals),
                  _lib.ptr(filled), _lib.ptr(self._filled_sum), B, n, T, float(self.gamma), B * T * self.world_size,
                  _lib.ptr(dq_tot),
                  _lib.ptr(self._stats), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer, [q_tot_eval], [dq_tot])
        return None

    def update(self, sample, sync=True):
        self.iterations += 1
        d = self._stacked(sample)
        info = self.callback.on_update_start(self.iterations, model=self.model, batch=d) or {}
        args = [d[k] for k in ('obs', 'actions', 'rewards', 'terminals', 'agent_mask', 'filled', 'state')]
        if d['avail'] is not None:
            args.append(d['avail'])
        self.optimizer.prepare()
        # the two collectives (sum(filled), gradient bucket) capture into the graph
        self._device_step(tuple(d['obs'].shape), self._device_update, *args)
        if self.scheduler is not None:
            self.scheduler.step()
        if sync:
            vals = self._info()
        if self.iterations % self.sync_frequency == 0:
            self.model.copy_target()
        if sync:
            self._finish_info(info, vals, model=self.model)
        return info

    def _info(self):
        """The logged values of the last update (reads the device statistics: one host synchronisation)."""
        s = self._stats.tolist()
        return {"learning_rate": self.optimizer.param_groups[0]['lr'], "loss_Q": s[0], "predictQ": s[1]}

"""VDAC and IAC learners - mirrors of xuance/torch/learners/multi_agent_rl/vdac_learner.py:15-147 and
iac_learner.py:157-289 (+ OnPolicyMultiAgentLearner) for one parameter-sharing group with Discrete actions.

update(sample): actor and critic forward over the packed rows -> the mixer (QMIX: K9 mix; VDN: inside K4V) ->
``xb_mappo_prepare`` -> [all-reduce of that 4-double block] -> ``xb_value_norm_update`` (use_value_norm) -> K4V fused
loss forward + backward (dlogits, dvalue, statistics into the bucket tail) -> torch backward into the flat bucket ->
[one all-reduce of gradient + statistics] -> K7 clip + Adam.  No host synchronisation until the info dict is built, so
the device half is capturable as a CUDA graph (``use_cuda_graph``), as in MAPPO_Learner.

The device buffers gather agent-major rows (agent k of sample b at k*B + b); the learner reorders them once to the
reference's packed (b, i, t) order, which is the row order K4V's value mixing reads.  With ``use_rnn`` the batch is B
whole episodes and the loss mask is agent_mask * filled.

The reference's recurrent VDAC pairs V_tot with the loss rows in a mismatched order (DESIGN.md section 4):
``config.vdac_rnn_reference_row_order = True`` reproduces it; the default pairs V_tot(b, t) with every agent's row of
step (b, t)."""
import torch

from ... import _lib
from ..utils import FusedAdam, allreduce_sum_, ValueNorm
from .learner import Learner

MIX_INDEPENDENT, MIX_VDN, MIX_EXTERNAL = 0, 1, 2


class VDAC_Learner(Learner):
    rank_suffix = False

    def __init__(self, config, agent_grouping, model, callback):
        super().__init__(config, model, callback)
        self.agent_grouping = agent_grouping
        self.group_keys = agent_grouping.group_keys
        if len(self.group_keys) != 1:
            raise NotImplementedError("%s: one parameter-sharing group" % type(self).__name__)
        self.agent_keys = agent_grouping.agent_keys
        self.n_agents = len(self.agent_keys)
        self.mix_mode = self._mix_mode(config)
        self.row_order = int(bool(getattr(config, "vdac_rnn_reference_row_order", False)) and self.use_rnn
                             and self.mix_mode != MIX_INDEPENDENT)
        self.use_global_state = (self.mix_mode == MIX_EXTERNAL) or getattr(config, "use_global_state", False)
        self.use_value_clip, self.value_clip_range = config.use_value_clip, config.value_clip_range
        self.use_huber_loss, self.huber_delta = config.use_huber_loss, config.huber_delta
        self.use_value_norm = config.use_value_norm
        self.vf_coef, self.ent_coef = config.vf_coef, config.ent_coef
        self._build_optimizer(config)
        self.value_normalizer = ({k: ValueNorm(1, device=self.device) for k in self.group_keys}
                                 if self.use_value_norm else None)
        self._prep = torch.zeros(4, dtype=torch.float64, device=self.device)
        self._stats = self._opt().bucket.tail[:8]
        self._scratch = _lib.scratch(self.device)
        if self.value_normalizer is not None:
            self._graph_tensors = [t for v in self.value_normalizer.values()
                                   for t in (v.running_mean, v.running_mean_sq, v.debiasing_term)]

    @staticmethod
    def _mix_mode(config):
        mixer = getattr(config, "mixer", "VDN")
        if mixer == "VDN":
            return MIX_VDN
        if mixer == "QMIX":
            return MIX_EXTERNAL
        raise NotImplementedError("VDAC_Learner: mixer %r is not supported (VDN or QMIX; IAC is the independent "
                                  "learner)" % (mixer,))

    def _build_optimizer(self, config):
        """LearnerMAS.build_optimizer (marl_learner.py:64-76): Adam(eps=1e-5) + LinearLR over every parameter."""
        self.optimizer = FusedAdam(self.model.parameters(), lr=self.learning_rate, eps=1e-5,
                                   weight_decay=getattr(config, "weight_decay", 0.0))
        self.scheduler = self._linear_lr(self.optimizer)

    def _opt(self):
        return self.optimizer

    def estimate_total_iterations(self):
        """marl_learner.py:203-214."""
        if getattr(self.config, "use_rnn", False):
            update_times = (self.config.running_steps // self.config.episode_length) // self.config.buffer_size
        else:
            update_times = self.config.running_steps // self.config.buffer_size
        return update_times * getattr(self.config, "n_epochs", 1) * getattr(self.config, "n_minibatch", 1)

    def _device_update(self, obs, actions, adv, values_old, returns, mask, avail=None, state=None):
        """vdac_learner.py:36-133 / iac_learner.py:190-264 on the device (static shapes, no host synchronisation).
        Rows are in (b, i, t) order; obs is [B*n, T, obs] with use_rnn, else [B*n, obs]."""
        n = self.n_agents
        R = actions.shape[0]
        T = obs.shape[1] if self.use_rnn else 1
        R_total = R * self.world_size
        logits = self.model.logits(obs)
        A = logits.shape[-1]
        logits = logits.reshape(-1, A).contiguous()
        v = self.model.values(obs).reshape(-1)
        if self.mix_mode == MIX_EXTERNAL:           # [B*T, n] per-step agent values -> V_tot [B*T] (K9 mix)
            v = self.model.values_tot(v.reshape(-1, n, T).transpose(1, 2), state).reshape(-1)
        v = v.contiguous()
        _lib.call("xb_mappo_prepare", _lib.ptr(mask), _lib.ptr(returns), R, _lib.ptr(self._prep),
                  _lib.ptr(self._scratch))
        if self.world_size > 1:
            allreduce_sum_(self._prep)                       # global sum(mask) and moments of the returns
        vn = None
        if self.value_normalizer is not None:
            norm = self.value_normalizer[self.group_keys[0]]
            norm.update_from_block(self._prep, R_total)
            vn = norm.mean_std
        dlogits, dvalue = torch.empty_like(logits), torch.empty_like(v)
        _lib.call("xb_vdac_loss_fwd_bwd", _lib.ptr(logits), _lib.ptr(avail), 0 if avail is None else avail.shape[1],
                  _lib.ptr(actions), _lib.ptr(adv), _lib.ptr(v), _lib.ptr(values_old), _lib.ptr(returns),
                  _lib.ptr(mask), _lib.ptr(vn), _lib.ptr(self._prep), R, A, n, T, self.mix_mode, self.row_order,
                  R_total, float(self.value_clip_range) if self.use_value_clip else 0.0,
                  float(self.huber_delta) if self.use_huber_loss else 0.0, float(self.vf_coef), float(self.ent_coef),
                  _lib.ptr(dlogits), _lib.ptr(dvalue), _lib.ptr(self._stats), _lib.ptr(self._scratch))
        self._optimizer_step(self._opt(), [logits, v], [dlogits, dvalue])
        return None

    def _args(self, sample):
        """The sample's agent-major device tensors in (b, i, t) row order."""
        st, n = sample['_stacked'], self.n_agents
        B = st['actions'].shape[0] // n
        packed = lambda x: x.reshape(n, B, *x.shape[1:]).transpose(0, 1).reshape(n * B, *x.shape[1:])
        mask = st['agent_mask'] * st['filled'] if self.use_rnn else st['agent_mask']
        rows = lambda x: packed(x).reshape(-1).contiguous()
        args = [packed(st['obs']).contiguous(), rows(st['actions']), rows(st['advantages']), rows(st['values']),
                rows(st['returns']), rows(mask)]
        avail = st.get('avail_actions') if self.use_actions_mask else None
        if avail is not None:
            avail = packed(avail).reshape(-1, avail.shape[-1]).contiguous()
        state = None
        if self.use_global_state and st.get('state') is not None:
            state = st['state'][:B].reshape(-1, st['state'].shape[-1]).contiguous()    # [B*T, S], row b*T + t
        return args + [avail, state]

    def update(self, sample, sync=True):
        self.iterations += 1
        args = self._args(sample)
        info = self.callback.on_update_start(self.iterations, model=self.model, batch=sample) or {}
        self._opt().prepare()
        self._device_step(tuple(args[0].shape), self._device_update, *args)
        self._step_scheduler()
        if sync:
            self._finish_info(info, self._info(self._stats.tolist()), model=self.model)
        return info

    def _step_scheduler(self):
        if self.scheduler is not None and self.use_linear_lr_decay:
            self.scheduler.step()

    def _info(self, s):
        g = self.group_keys[0]
        vals = {f"{g}/actor_loss": s[0], f"{g}/critic_loss": s[1], f"{g}/entropy": s[2], f"{g}/predict_value": s[3]}
        if self.use_grad_clip:
            vals["gradient_norm"] = float(self.optimizer.grad_norm.item())
        vals.update({"learning_rate": self.optimizer.param_groups[0]['lr'], "loss": s[4]})
        return vals


class IAC_Learner(VDAC_Learner):
    """iac_learner.py:157-289: per-agent critics (no mixer), one Adam + LinearLR per group; the LinearLR steps every
    update whether or not use_linear_lr_decay is set (iac_learner.py:265-266)."""

    @staticmethod
    def _mix_mode(config):
        return MIX_INDEPENDENT

    def _build_optimizer(self, config):
        g = self.group_keys[0]
        opt = FusedAdam(self.model.parameters(), lr=self.learning_rate, eps=1e-5,
                        weight_decay=getattr(config, "weight_decay", 0.0))
        self.optimizer = {g: opt}
        self.scheduler = {g: self._linear_lr(opt)}

    def _opt(self):
        return self.optimizer[self.group_keys[0]]

    def _step_scheduler(self):
        self.scheduler[self.group_keys[0]].step()

    def _info(self, s):
        g = self.group_keys[0]
        vals = {}
        if self.use_grad_clip:
            vals["gradient_norm"] = float(self._opt().grad_norm.item())
        vals.update({f"{g}/actor_loss": s[0], f"{g}/critic_loss": s[1], f"{g}/entropy": s[2],
                     f"{g}/total_loss": s[4], f"{g}/predict_value": s[3],
                     f"{g}/learning_rate": self._opt().param_groups[0]['lr']})
        return vals

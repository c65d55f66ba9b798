"""MAPPO learner - mirror of xuance/torch/learners/multi_agent_rl/mappo_learner.py:14-149 (+ OnPolicyMultiAgentLearner,
base/marl_learner.py:18-76, 184-302) for one parameter-sharing group of feed-forward agents with Discrete actions.

update(sample): actor and critic forward over the packed rows -> ``xb_mappo_prepare`` (sum of the agent mask, moments
of the returns) -> [all-reduce of that 4-double block] -> ``xb_value_norm_update`` (use_value_norm) -> K4M fused loss
forward + backward (dlogits, dvalue, statistics into the bucket tail) -> torch backward into the flat bucket ->
[one all-reduce of gradient + statistics] -> K7 clip + Adam.  No host synchronisation until the info dict is built, so
the device half is capturable as a CUDA graph (``use_cuda_graph``).

With ``use_rnn`` the batch is B whole episodes: the actor and the critic run over the [B*n, T] sequences from zero states
(the GRU recurrence on K13, captured with the rest), and K4M runs over the R = B*n*T rows with mask = agent_mask * filled
(modules/outputs.py:133-143 ``valid_mask``).  The ValueNorm update and predict_value see every row, masked or not, as in
the reference."""
import torch

from ... import _lib
from ..utils import FusedAdam, allreduce_sum_, ValueNorm
from .learner import Learner


class MAPPO_Learner(Learner):
    rank_suffix = False

    def __init__(self, config, agent_grouping, model, callback):
        super().__init__(config, model, callback)
        self.use_parameter_sharing = getattr(config, "use_parameter_sharing", True)
        self.agent_grouping = agent_grouping
        self.group_keys = agent_grouping.group_keys
        if len(self.group_keys) != 1:
            raise NotImplementedError("MAPPO_Learner: one parameter-sharing group")
        self.agent_keys = agent_grouping.agent_keys
        self.n_agents = len(self.agent_keys)
        self.clip_range = config.clip_range
        self.use_global_state = getattr(config, "use_global_state", False)
        self.use_value_clip, self.value_clip_range = config.use_value_clip, config.value_clip_range
        self.use_huber_loss, self.huber_delta = config.use_huber_loss, config.huber_delta
        self.use_value_norm = config.use_value_norm
        self.use_rnn = getattr(config, "use_rnn", False)
        self.vf_coef, self.ent_coef = config.vf_coef, config.ent_coef
        # LearnerMAS.build_optimizer (marl_learner.py:64-76): Adam(eps=1e-5) + LinearLR, stepped only with decay on
        self.optimizer = FusedAdam(self.model.parameters(), lr=self.learning_rate, eps=1e-5,
                                   weight_decay=getattr(config, "weight_decay", 0.0))
        self.scheduler = self._linear_lr(self.optimizer)
        self.value_normalizer = ({k: ValueNorm(1, device=self.device) for k in self.group_keys}
                                 if self.use_value_norm else None)
        self._prep = torch.zeros(4, dtype=torch.float64, device=self.device)
        self._stats = self.optimizer.bucket.tail[:8]
        self._scratch = _lib.scratch(self.device)
        if self.value_normalizer is not None:
            self._graph_tensors = [t for v in self.value_normalizer.values()
                                   for t in (v.running_mean, v.running_mean_sq, v.debiasing_term)]

    def estimate_total_iterations(self):
        """marl_learner.py:203-214."""
        if getattr(self.config, "use_rnn", False):
            update_times = (self.config.running_steps // self.config.episode_length) // self.config.buffer_size
        else:
            update_times = self.config.running_steps // self.config.buffer_size
        return update_times * getattr(self.config, "n_epochs", 1) * getattr(self.config, "n_minibatch", 1)

    def _device_update(self, obs, actions, old_logp, adv, values_old, returns, mask, avail=None, state=None):
        """mappo_learner.py:41-137 on the device (static shapes, no host synchronisation)."""
        R = actions.shape[0]
        R_total = R * self.world_size
        logits = self.model.logits(obs)
        A = logits.shape[-1]
        logits = logits.reshape(-1, A).contiguous()             # [B*n, T, A] -> rows (recurrent batches)
        v_pred = self.model.values(obs, state if self.use_global_state else None).reshape(-1).contiguous()
        _lib.call("xb_mappo_prepare", _lib.ptr(mask), _lib.ptr(returns), R, _lib.ptr(self._prep),
                  _lib.ptr(self._scratch))
        if self.world_size > 1:
            allreduce_sum_(self._prep)                       # global sum(mask) and moments of the returns
        vn = None
        if self.value_normalizer is not None:
            norm = self.value_normalizer[self.group_keys[0]]
            norm.update_from_block(self._prep, R_total)
            vn = norm.mean_std
        dlogits, dvalue = torch.empty_like(logits), torch.empty_like(v_pred)
        _lib.call("xb_mappo_loss_fwd_bwd", _lib.ptr(logits), _lib.ptr(avail), 0 if avail is None else avail.shape[1],
                  _lib.ptr(actions), _lib.ptr(old_logp), _lib.ptr(adv), _lib.ptr(v_pred), _lib.ptr(values_old),
                  _lib.ptr(returns), _lib.ptr(mask), _lib.ptr(vn), _lib.ptr(self._prep), R, A, R_total,
                  float(self.clip_range), float(self.value_clip_range) if self.use_value_clip else 0.0,
                  float(self.huber_delta) if self.use_huber_loss else 0.0, float(self.vf_coef), float(self.ent_coef),
                  _lib.ptr(dlogits), _lib.ptr(dvalue), _lib.ptr(self._stats), _lib.ptr(self._scratch))
        self._optimizer_step(self.optimizer, [logits, v_pred], [dlogits, dvalue])
        return None

    def _args(self, sample):
        st = sample['_stacked']
        if self.use_rnn:            # [B*n, T] fields -> B*n*T rows; the loss mask is agent_mask * filled
            f = lambda k: st[k].reshape(-1)
            args = [st['obs'], f('actions'), f('log_pi_old'), f('advantages'), f('values'), f('returns'),
                    (st['agent_mask'] * st['filled']).reshape(-1)]
        else:
            args = [st['obs'], st['actions'], st['log_pi_old'], st['advantages'], st['values'], st['returns'],
                    st['agent_mask']]
        avail = st.get('avail_actions') if self.use_actions_mask else None
        state = st.get('state') if self.use_global_state else None
        if avail is not None:
            avail = avail.reshape(-1, avail.shape[-1]).contiguous()
        return [a.contiguous() for a in args] + [avail, state]

    def update(self, sample, sync=True):
        self.iterations += 1
        args = self._args(sample)
        info = self.callback.on_update_start(self.iterations, model=self.model, batch=sample) or {}
        self.optimizer.prepare()
        self._device_step(tuple(args[0].shape), self._device_update, *args)
        if self.scheduler is not None and self.use_linear_lr_decay:
            self.scheduler.step()
        if sync:
            s = self._stats.tolist()
            g = self.group_keys[0]
            vals = {f"{g}/actor_loss": s[0], f"{g}/critic_loss": s[1], f"{g}/entropy": s[2], f"{g}/predict_value": s[3]}
            if self.use_grad_clip:
                vals["gradient_norm"] = float(self.optimizer.grad_norm.item())
            vals.update({"learning_rate": self.optimizer.param_groups[0]['lr'], "loss": s[4]})
            self._finish_info(info, vals, model=self.model)
        return info

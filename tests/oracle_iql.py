"""torch-CPU float64 oracle of one IQL_Learner update (iql_learner.py:37-142 for one shared group of GRU agents, with
q_eval keeping its graph and the next-step masks sliced on the time axis, DESIGN.md section 4): the same parameters as a
product MixingQNetwork, the GRU as torch's nn.GRU, the loss in the reference's own expressions (tests/iql_refs.py).
``update`` runs a whole update (Adam with eps 1e-5, optional clip_grad_norm_, LinearLR, then the target sync every
``sync_frequency`` updates) and returns the reference's info dict."""
from copy import deepcopy

import numpy as np
import torch

import iql_refs as R


def build_model(n, obs_dim, A, hid, device):
    """A product MixingQNetwork built as IQL_Agents builds it (K13 GRU agents of width hid, Q head [hid], the
    IndependentMixer); on the CPU it holds the parameters for the oracle and for a strict reference state_dict load."""
    import torch.nn as nn
    from xuance_b200.common import AgentGrouping, Discrete
    from xuance_b200.torch.rl_models import (AgentFeatureEncoder, Basic_RNN_K13, DiscreteActionValueCritic,
                                             IndependentMixer, MixingQNetwork)
    keys = [f"agent_{i}" for i in range(n)]
    rep = Basic_RNN_K13(input_shape=(obs_dim,), initialize=nn.init.orthogonal_, activation=nn.ReLU, device=device,
                        fc_hidden_sizes=[hid], recurrent_hidden_size=hid)
    q = DiscreteActionValueCritic(AgentFeatureEncoder(rep), Discrete(A), [hid], None, nn.init.orthogonal_, nn.ReLU,
                                  device)
    grouping = AgentGrouping.shared(keys)
    model = MixingQNetwork(grouping, nn.ModuleDict({"shared": q}), IndependentMixer(), use_rnn=True,
                           device=device).to(device)
    return keys, grouping, model


class IQLOracle:
    def __init__(self, model, double_q=True, gamma=0.99, learning_rate=7e-4, end_factor_lr_decay=0.5, total_iters=1,
                 sync_frequency=2, use_actions_mask=True, grad_clip_norm=None):
        self.m = deepcopy(model).cpu().double()
        self.g = self.m.group_keys[0]
        self.keys = self.m.agent_keys
        self.double_q, self.gamma, self.use_actions_mask = double_q, gamma, use_actions_mask
        self.grad_clip_norm = grad_clip_norm
        self.optimizer = torch.optim.Adam(self.m.parameters_model, lr=learning_rate, eps=1e-5)
        self.scheduler = torch.optim.lr_scheduler.LinearLR(self.optimizer, start_factor=1.0,
                                                           end_factor=end_factor_lr_decay, total_iters=total_iters)
        self.sync_frequency, self.iterations = sync_frequency, 0

    def _q(self, obs, target):
        """obs [B, n, T+1, o] -> q [B, n, T+1, A] from a zero state."""
        net = (self.m.target_individual_q_networks if target else self.m.individual_q_networks)[self.g]
        rep = net.representation.obs_representation
        B, n, T1, _ = obs.shape
        y, _ = rep.rnn(rep.mlp(obs.reshape(B * n, T1, -1)))
        return net.critic_head(y).reshape(B, n, T1, -1)

    def _batch(self, s):
        st = lambda k: torch.from_numpy(np.stack([np.asarray(s[k][a]) for a in self.keys], axis=1))
        b = {k: st(k).double() for k in ("obs", "actions", "rewards", "terminals", "agent_mask")}
        b["avail"] = st("avail_actions").to(torch.uint8) if self.use_actions_mask else None
        b["filled"] = torch.from_numpy(np.asarray(s["filled"])).double()
        return b

    def forward(self, s):
        b = self._batch(s)
        q_all = self._q(b["obs"], False)
        with torch.no_grad():
            q_tgt = self._q(b["obs"], True)
        return R.forward(q_all, q_tgt, b["actions"], b["rewards"], b["terminals"], b["agent_mask"], b["filled"],
                         b["avail"], self.double_q, self.gamma)

    def losses(self, s):
        loss, pq = self.forward(s)[:2]
        return [loss.item(), pq.item()]

    def grads(self, s):
        self.m.zero_grad()
        self.forward(s)[0].backward()
        names = {id(p): k for k, p in self.m.named_parameters()}
        return {names[id(p)]: (p.grad if p.grad is not None else torch.zeros_like(p)) for p in self.m.parameters_model}

    def update(self, s):
        self.iterations += 1
        loss, pq = self.forward(s)[:2]
        self.optimizer.zero_grad()
        loss.backward()
        if self.grad_clip_norm is not None:
            torch.nn.utils.clip_grad_norm_(self.m.parameters_model, self.grad_clip_norm)
        self.optimizer.step()
        self.scheduler.step()
        info = {f"{self.g}/learning_rate": self.optimizer.param_groups[0]["lr"], f"{self.g}/loss_Q": loss.item(),
                f"{self.g}/predictQ": pq.item()}
        if self.iterations % self.sync_frequency == 0:
            self.m.copy_target()
        return info

"""torch-CPU float64 oracle of one QTRAN_Learner update (qtran_learner.py:199-371 for one shared group of GRU agents):
the same parameters as a product QTranMixingNetwork, the GRU as torch's nn.GRU, every step in the reference's own
expressions (tests/qtran_refs.py).  ``losses`` gives the logged values; ``grads`` the gradient of every parameter of
``parameters_model``, by name; ``update`` runs a whole update (Adam with eps 1e-5 and LinearLR, as
marl_learner.py:64-76, then the target sync every ``sync_frequency`` updates) and returns the reference's info dict."""
from copy import deepcopy

import numpy as np
import torch

import qtran_refs as R


INFO_KEYS = ("loss_td", "loss_opt", "loss_nopt", "loss", "Q_joint")


def build_model(agent, n, obs_dim, A, S, hid, qhid, device):
    """A product QTranMixingNetwork built as QTRAN_Agents builds it (K13 GRU agents of width hid, Q_jt / V_jt of width
    qhid); on the CPU it holds the parameters for the oracle and for a strict reference state_dict load."""
    import torch.nn as nn
    from xuance_b200.common import AgentGrouping, Discrete
    from xuance_b200.torch.rl_models import (AgentFeatureEncoder, Basic_RNN_K13, DiscreteActionValueCritic, VDN_mixer,
                                             QTRAN_Base, QTRAN_Alt, QTranMixingNetwork)
    keys = [f"agent_{i}" for i in range(n)]
    rep = Basic_RNN_K13(input_shape=(obs_dim,), initialize=nn.init.orthogonal_, activation=nn.ReLU, device=device,
                        fc_hidden_sizes=[hid], recurrent_hidden_size=hid)
    q = DiscreteActionValueCritic(AgentFeatureEncoder(rep), Discrete(A), [hid], None, nn.init.orthogonal_, nn.ReLU,
                                  device)
    head = (QTRAN_Base if agent == "QTRAN_base" else QTRAN_Alt)(S, {k: Discrete(A) for k in keys}, qhid, n, hid, True,
                                                                   device)
    grouping = AgentGrouping.shared(keys)
    model = QTranMixingNetwork(grouping, nn.ModuleDict({"shared": q}), VDN_mixer(), head, use_rnn=True,
                               device=device).to(device)
    return keys, grouping, model


class QTRANOracle:
    def __init__(self, model, double_q=True, gamma=0.99, lambda_opt=1.0, lambda_nopt=1.0, learning_rate=7e-4,
                 end_factor_lr_decay=0.5, total_iters=1, sync_frequency=2):
        self.m = deepcopy(model).cpu().double()
        self.g = self.m.group_keys[0]
        self.keys = self.m.agent_keys
        self.double_q, self.gamma, self.lo, self.ln = double_q, gamma, lambda_opt, lambda_nopt
        self.optimizer = torch.optim.Adam(self.m.parameters_model, lr=learning_rate, eps=1e-5)
        self.scheduler = torch.optim.lr_scheduler.LinearLR(self.optimizer, start_factor=1.0,
                                                           end_factor=end_factor_lr_decay, total_iters=total_iters)
        self.sync_frequency, self.iterations = sync_frequency, 0

    def _agents(self, obs, target):
        """obs [B, n, T+1, o] -> (q [B, n, T+1, A], h [B, n, T+1, H]) from a zero state."""
        net = (self.m.target_individual_q_networks if target else self.m.individual_q_networks)[self.g]
        rep = net.representation.obs_representation
        B, n, T1, _ = obs.shape
        y, _ = rep.rnn(rep.mlp(obs.reshape(B * n, T1, -1)))
        q = net.critic_head(y)
        return q.reshape(B, n, T1, -1), y.reshape(B, n, T1, -1)

    def _batch(self, s):
        st = lambda k: torch.from_numpy(np.stack([np.asarray(s[k][a]) for a in self.keys], axis=1))
        b = {k: st(k).double() for k in ("obs", "actions", "rewards", "terminals", "agent_mask")}
        b["avail"] = st("avail_actions").to(torch.uint8)
        b["filled"] = torch.from_numpy(np.asarray(s["filled"])).double()
        b["state"] = torch.from_numpy(np.asarray(s["state"])).double()
        return b

    def loss(self, s):
        b = self._batch(s)
        net, tnet = self.m.qtran_net, self.m.target_qtran_net
        q_all, h = self._agents(b["obs"], False)
        with torch.no_grad():
            q_tgt, h_tgt = self._agents(b["obs"], True)
        greedy, nxt = R.select_ref(q_all.detach(), q_tgt, b["avail"], self.double_q)
        enc = lambda m_, *a: R.encode_ref(m_.mode, *a, m_.action_encoding[0].weight, m_.action_encoding[0].bias,
                                          m_.action_encoding[2].weight, m_.action_encoding[2].bias)
        st, mask = b["state"], b["agent_mask"]
        B, T = mask.shape[0], mask.shape[2]
        qjt = net.Q_jt(enc(net, st, 0, h, mask, b["actions"]))
        v = net.V_jt(st[:, :-1].reshape(B * T, -1))
        with torch.no_grad():
            qjt_g = net.Q_jt(enc(net, st, 0, h, mask, greedy))
            qjt_n = tnet.Q_jt(enc(tnet, st, 1, h_tgt, mask, nxt))
        return R.loss_ref(net.mode, q_all, b["actions"], greedy, nxt, mask, b["filled"], b["rewards"].float(),
                          b["terminals"], qjt.reshape(-1) if net.mode == R.BASE else qjt, qjt_g, qjt_n, v.reshape(-1),
                          self.gamma, self.lo, self.ln)

    def losses(self, s):
        return self.loss(s)[1].tolist()

    def grads(self, s):
        self.m.zero_grad()
        self.loss(s)[0].backward()
        names = {id(p): k for k, p in self.m.named_parameters()}
        return {names[id(p)]: (p.grad if p.grad is not None else torch.zeros_like(p)) for p in self.m.parameters_model}

    def update(self, s):
        self.iterations += 1
        loss, stats = self.loss(s)
        self.optimizer.zero_grad()
        loss.backward()
        self.optimizer.step()
        self.scheduler.step()
        if self.iterations % self.sync_frequency == 0:
            self.m.copy_target()
        info = dict(zip(INFO_KEYS, stats.tolist()))
        info["learning_rate"] = self.optimizer.param_groups[0]["lr"]
        return info

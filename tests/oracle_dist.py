"""Torch-CPU oracle of the C51 / QR-DQN stacks, built on ``oracle/`` (its ``mlp`` builder) and independent of the
product's classes; pinned to tests/golden/c51_qrdqn_update.npz (generated from the unmodified reference).

* ``DistModelOracle``   C51DeepQNetwork / QRDeepQNetwork over a Basic_MLP encoder, or a Basic_CNN one with ``pixels=True``
                        (deep_q_network.py:146-325, q_head.py:83-123), with the reference's parameter names (C51's
                        ``supports`` included, as a CPU-built reference saves it);
* ``DistLearnerOracle`` c51_learner.py:27-81 and qrdqn_learner.py:29-77 with torch autograd, torch.optim.Adam (eps 1e-5) and
                        LinearLR."""
import copy
import os
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.nets import mlp, PoolEncoderQ  # noqa: E402


def _box(**children):
    m = nn.Module()
    for k, v in children.items():
        setattr(m, k, v)
    return m


class DistModelOracle(nn.Module):
    def __init__(self, algo, obs_dim, n_actions, n_atoms, rep_hidden=(32,), q_hidden=(32,), v_min=-10, v_max=10,
                 act=nn.ReLU, pixels=False):
        """``pixels=True``: the Basic_CNN encoder of the Atari configs on 84x84x4 uint8 frames (``obs_dim`` unused)."""
        super().__init__()
        init = nn.init.orthogonal_
        self.algo, self.n_actions, self.n_atoms, self.pixels = algo, n_actions, n_atoms, pixels
        if pixels:
            self.representation, feat = PoolEncoderQ(), 64
        else:
            self.representation = _box(model=mlp([obs_dim, *rep_hidden], act=act, last_act=True, init=init))
            feat = rep_hidden[-1]
        self.target_representation = copy.deepcopy(self.representation)
        self.eval_Z_head = _box(model=mlp([feat, *q_hidden, n_actions * n_atoms], act=act, init=init))
        self.target_Z_head = copy.deepcopy(self.eval_Z_head)
        if algo == "c51":
            self.v_min, self.v_max = v_min, v_max
            self.supports = nn.Parameter(torch.linspace(v_min, v_max, n_atoms), requires_grad=False)
            self.delta_z = (v_max - v_min) / (n_atoms - 1)

    def _z(self, rep, head, obs):
        z = head.model(rep(obs) if self.pixels else rep.model(obs)).view(-1, self.n_actions, self.n_atoms)
        return torch.softmax(z, dim=-1) if self.algo == "c51" else z

    def _q(self, z):
        return (self.supports * z).sum(-1) if self.algo == "c51" else z.mean(dim=-1)

    def forward(self, obs):
        z = self._z(self.representation, self.eval_Z_head, obs)
        return self._q(z).argmax(dim=-1), z

    def target(self, obs):
        z = self._z(self.target_representation, self.target_Z_head, obs)
        return self._q(z).argmax(dim=-1), z

    def copy_target(self):
        for src, dst in ((self.representation, self.target_representation), (self.eval_Z_head, self.target_Z_head)):
            for ep, tp in zip(src.parameters(), dst.parameters()):
                tp.data.copy_(ep)


class DistLearnerOracle:
    def __init__(self, model, lr=1e-3, gamma=0.99, sync_frequency=100, use_grad_clip=False, grad_clip_norm=0.5,
                 end_factor_lr_decay=1.0, total_iters=1):
        self.model = model
        self.optimizer = torch.optim.Adam(model.parameters(), lr, eps=1e-5)
        self.scheduler = torch.optim.lr_scheduler.LinearLR(self.optimizer, start_factor=1.0,
                                                           end_factor=end_factor_lr_decay, total_iters=total_iters)
        self.gamma, self.sync_frequency = gamma, sync_frequency
        self.use_grad_clip, self.grad_clip_norm = use_grad_clip, grad_clip_norm
        self.iterations = 0

    def loss(self, obs, act, nxt, rew, ter):
        m = self.model
        N = m.n_atoms
        _, evalZ = m(obs)
        targetA, targetZ = m.target(nxt)
        a = act.reshape(-1, 1, 1).long()
        cur = evalZ.gather(1, a.expand([-1, -1, N])).squeeze(1)
        tgt = targetZ.gather(1, targetA.reshape([-1, 1, 1]).expand([-1, -1, N])).squeeze(1)
        if m.algo == "c51":
            tgt = tgt.detach()
            nxt_sup = (rew.unsqueeze(1) + self.gamma * m.supports * (1 - ter.unsqueeze(1))).clamp(m.v_min, m.v_max)
            proj = 1 - (nxt_sup.unsqueeze(-1) - m.supports.unsqueeze(0)).abs() / m.delta_z
            tgt = torch.bmm(tgt.unsqueeze(1), proj.clamp(0, 1)).squeeze(1)
            return -(tgt * torch.log(cur + 1e-8)).sum(1).mean()
        tgt = rew.unsqueeze(1) + self.gamma * tgt * (1 - ter.unsqueeze(1))
        return nn.functional.mse_loss(tgt.detach(), cur)

    def update(self, **s):
        self.iterations += 1
        t = lambda k, dt=None: torch.as_tensor(s[k], dtype=dt)
        loss = self.loss(t('obs'), t('actions'), t('obs_next'), t('rewards'), t('terminals', torch.float))
        self.optimizer.zero_grad()
        loss.backward()
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(self.model.parameters(), self.grad_clip_norm)
        self.optimizer.step()
        self.scheduler.step()
        if self.iterations % self.sync_frequency == 0:
            self.model.copy_target()
        return {"Qloss": loss.item(), "learning_rate": self.optimizer.param_groups[0]['lr']}

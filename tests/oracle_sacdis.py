"""Torch-CPU oracle of the SAC-Discrete stack, built on ``oracle/`` (its ``mlp`` builder) and independent of the product's
classes; pinned to tests/golden/sacdis_update.npz (generated from the unmodified reference).

* ``SACDISModelOracle``   SoftActorCriticDiscrete(CategoricalActor, TwinDiscreteActionValueCritic) over Basic_MLP encoders
                          (actor_critic.py:162-214, twin_critics.py:65-117), with the reference's parameter names;
* ``SACDISLearnerOracle`` sacdis_learner.py:12-129 with torch autograd, torch.optim.Adam and LinearLR."""
import copy
import os
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.nets import mlp  # noqa: E402


def _box(**children):
    m = nn.Module()
    for k, v in children.items():
        setattr(m, k, v)
    return m


class SACDISModelOracle(nn.Module):
    def __init__(self, obs_dim, n_actions, rep_hidden=(32,), actor_hidden=(32,), critic_hidden=(32,)):
        super().__init__()
        init = nn.init.orthogonal_
        enc = lambda: _box(model=mlp([obs_dim, *rep_hidden], last_act=True, init=init))
        self.actor = _box(representation=enc(),
                          actor_head=_box(logits=mlp([rep_hidden[-1], *actor_hidden, n_actions], init=init)))
        head = lambda: _box(q_value=mlp([rep_hidden[-1], *critic_hidden, n_actions], init=init))
        self.critic = _box(representation_1=enc(), representation_2=enc(), critic_head_1=head(), critic_head_2=head())
        self.target_critic = copy.deepcopy(self.critic)
        self.n_actions = n_actions

    def _probs(self, obs):
        p = torch.distributions.Categorical(logits=self.actor.actor_head.logits(self.actor.representation.model(obs))).probs
        return p, torch.log(p + (p == 0.0).float() * 1e-8)

    @staticmethod
    def _q(critic, obs):
        return (critic.critic_head_1.q_value(critic.representation_1.model(obs)),
                critic.critic_head_2.q_value(critic.representation_2.model(obs)))

    def Qpolicy(self, obs):
        p, lp = self._probs(obs)
        q1, q2 = self._q(self.critic, obs)
        return p, lp, q1, q2

    def Qtarget(self, obs):
        p, lp = self._probs(obs)
        q1, q2 = self._q(self.target_critic, obs)
        return p, lp, torch.min(q1, q2)

    def Qaction(self, obs):
        return self._q(self.critic, obs)

    def soft_update(self, tau):
        for ep, tp in zip(self.critic.parameters(), self.target_critic.parameters()):
            tp.data.mul_(1 - tau)
            tp.data.add_(tau * ep.data)


class SACDISLearnerOracle:
    def __init__(self, model, lr_actor=1e-3, lr_critic=1e-3, tau=0.005, gamma=0.99, alpha=0.2, auto_alpha=False,
                 use_grad_clip=False, grad_clip_norm=0.5, end_factor_lr_decay=1.0, total_iters=1):
        self.model = model
        self.opt_a = torch.optim.Adam(model.actor.parameters(), lr_actor)
        self.opt_c = torch.optim.Adam(model.critic.parameters(), lr_critic)
        mk = lambda o: torch.optim.lr_scheduler.LinearLR(o, start_factor=1.0, end_factor=end_factor_lr_decay,
                                                         total_iters=total_iters)
        self.sch_a, self.sch_c = mk(self.opt_a), mk(self.opt_c)
        self.tau, self.gamma, self.alpha = tau, gamma, alpha
        self.auto = auto_alpha
        self.use_grad_clip, self.grad_clip_norm = use_grad_clip, grad_clip_norm
        if auto_alpha:
            self.target_entropy = -float(model.n_actions)
            self.log_alpha = nn.Parameter(torch.zeros(1, requires_grad=True))
            self.alpha = self.log_alpha.exp()
            self.opt_alpha = torch.optim.Adam([self.log_alpha], lr=lr_actor)

    def update(self, **s):
        obs = torch.as_tensor(s['obs'])
        act = torch.as_tensor(s['actions']).unsqueeze(-1)
        nxt, rew = torch.as_tensor(s['obs_next']), torch.as_tensor(s['rewards']).unsqueeze(-1)
        ter = torch.as_tensor(s['terminals'], dtype=torch.float).reshape([-1, 1])
        p, log_pi, q1, q2 = self.model.Qpolicy(obs)
        model_q = torch.min(q1, q2)
        p_loss = (p * (self.alpha * log_pi - model_q)).sum(dim=1).mean()
        self.opt_a.zero_grad()
        p_loss.backward()
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(self.model.actor.parameters(), self.grad_clip_norm)
        self.opt_a.step()
        aq1, aq2 = self.model.Qaction(obs)
        aq1, aq2 = aq1.gather(1, act.long()), aq2.gather(1, act.long())
        p_next, log_pi_next, target_q = self.model.Qtarget(nxt)
        target_q = (p_next * (target_q - self.alpha * log_pi_next)).sum(dim=1).unsqueeze(-1)
        backup = rew + (1 - ter) * self.gamma * target_q
        q_loss = nn.functional.mse_loss(aq1, backup.detach()) + nn.functional.mse_loss(aq2, backup.detach())
        self.opt_c.zero_grad()
        q_loss.backward()
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(self.model.critic.parameters(), self.grad_clip_norm)
        self.opt_c.step()
        info = {"Qloss": q_loss.item(), "Ploss": p_loss.item(), "Qvalue": model_q.mean().item()}
        if self.auto:
            alpha_loss = -(self.log_alpha * (log_pi + self.target_entropy).detach()).mean()
            self.opt_alpha.zero_grad()
            alpha_loss.backward()
            self.opt_alpha.step()
            self.alpha = self.log_alpha.exp()
            info.update(alpha_loss=alpha_loss.item(), alpha=self.alpha.item())
        self.sch_a.step()
        self.sch_c.step()
        self.model.soft_update(self.tau)
        info.update(actor_lr=self.opt_a.param_groups[0]['lr'], critic_lr=self.opt_c.param_groups[0]['lr'])
        return info

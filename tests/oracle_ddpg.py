"""Torch-CPU oracle of the DDPG / TD3 stacks, built on ``oracle/`` (its ``mlp`` builder) and independent of the product's
classes; pinned to tests/golden/ddpg_td3_update.npz (generated from the unmodified reference).

* ``DDPGModelOracle``   DeterministicActorCritic / TwinDelayedActorCritic over Basic_MLP encoders (actor_critic.py:217-319,
                        deterministic_actors.py, base_critics.py:47-88, twin_critics.py:11-62) with the reference's
                        parameter names; TD3's target-policy noise is supplied by the caller;
* ``DDPGLearnerOracle`` ddpg_learner.py:12-94 and td3_learner.py:12-100 with torch autograd, torch.optim.Adam and LinearLR."""
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


class DDPGModelOracle(nn.Module):
    def __init__(self, obs_dim, act_dim, low, high, twin, rep_hidden=(32,), actor_hidden=(32,), critic_hidden=(32,),
                 sigma=0.2, noise_clip=0.5, act=nn.ReLU):
        """``rep_hidden=()`` is the Basic_Identical representation."""
        super().__init__()
        init = nn.init.orthogonal_
        feat = rep_hidden[-1] if rep_hidden else obs_dim
        enc = lambda: _box(model=mlp([obs_dim, *rep_hidden], act=act, last_act=True, init=init))
        head = nn.Sequential(*mlp([feat, *actor_hidden, act_dim], act=act, init=init), nn.Tanh())
        self.actor = _box(representation=enc(), actor_head=_box(model=head))
        value = lambda: _box(values=mlp([feat + act_dim, *critic_hidden, 1], act=act, init=init))
        if twin:
            self.critic = _box(representation_1=enc(), representation_2=enc(), critic_head_1=value(),
                               critic_head_2=value())
        else:
            self.critic = _box(representation=enc(), critic_head=value())
        self.target_actor = copy.deepcopy(self.actor)
        self.target_critic = copy.deepcopy(self.critic)
        self.twin = twin
        self.low, self.high = torch.as_tensor(low), torch.as_tensor(high)
        self.sigma, self.noise_clip = sigma, noise_clip

    @staticmethod
    def _act(actor, obs):
        return actor.actor_head.model(actor.representation.model(obs))

    def _q(self, critic, obs, act):
        v = lambda r, h: h.values(torch.concat([r.model(obs), act], dim=-1)).squeeze(-1)
        if self.twin:
            return v(critic.representation_1, critic.critic_head_1), v(critic.representation_2, critic.critic_head_2)
        return v(critic.representation, critic.critic_head)

    def act(self, obs):
        return self._act(self.actor, obs)

    def Qaction(self, obs, act):
        return self._q(self.critic, obs, act)

    def Qtarget(self, obs, noise=None):
        ta = self._act(self.target_actor, obs)
        if not self.twin:
            return self._q(self.target_critic, obs, ta)
        n = (noise * self.sigma).clamp(-self.noise_clip, self.noise_clip)
        ta = torch.maximum(torch.minimum(ta + n, self.high), self.low)
        return torch.minimum(*self._q(self.target_critic, obs, ta))

    def Qpolicy(self, obs):
        q = self._q(self.critic, obs, self._act(self.actor, obs))
        return (q[0] + q[1]) / 2.0 if self.twin else q

    def soft_update(self, tau):
        for src, dst in ((self.actor, self.target_actor), (self.critic, self.target_critic)):
            for ep, tp in zip(src.parameters(), dst.parameters()):
                tp.data.mul_(1 - tau)
                tp.data.add_(tau * ep.data)


class DDPGLearnerOracle:
    def __init__(self, model, lr_actor=1e-3, lr_critic=1e-3, tau=0.005, gamma=0.99, actor_update_delay=1,
                 use_grad_clip=False, grad_clip_norm=0.5, end_factor_lr_decay=1.0, total_iters=1):
        self.model = model
        self.opt_a = torch.optim.Adam(model.actor.parameters(), lr_actor)
        self.opt_c = torch.optim.Adam(model.critic.parameters(), lr_critic)
        mk = lambda o: torch.optim.lr_scheduler.LinearLR(o, start_factor=1.0, end_factor=end_factor_lr_decay,
                                                         total_iters=total_iters)
        self.sch_a, self.sch_c = mk(self.opt_a), mk(self.opt_c)
        self.tau, self.gamma, self.delay = tau, gamma, actor_update_delay
        self.use_grad_clip, self.grad_clip_norm = use_grad_clip, grad_clip_norm
        self.iterations = 0

    def _step(self, opt, module, loss):
        opt.zero_grad()
        loss.backward()
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(module.parameters(), self.grad_clip_norm)
        opt.step()

    def update(self, noise_next=None, **s):
        self.iterations += 1
        m = self.model
        obs, act = torch.as_tensor(s['obs']), torch.as_tensor(s['actions'])
        nxt, rew = torch.as_tensor(s['obs_next']), torch.as_tensor(s['rewards'])
        ter = torch.as_tensor(s['terminals'], dtype=torch.float)
        mse = nn.functional.mse_loss
        info = {}
        if m.twin:
            qa, qb = m.Qaction(obs, act)
            next_q = m.Qtarget(nxt, torch.as_tensor(noise_next))
            target_q = rew + self.gamma * (1 - ter) * next_q
            q_loss = mse(qa, target_q.detach()) + mse(qb, target_q.detach())
            self._step(self.opt_c, m.critic, q_loss)
            self.sch_c.step()
            if self.iterations % self.delay == 0:
                p_loss = -m.Qpolicy(obs).mean()
                self._step(self.opt_a, m.actor, p_loss)
                self.sch_a.step()
                m.soft_update(self.tau)
                info["Ploss"] = p_loss.item()
            info.update(Qloss=q_loss.item(), QvalueA=qa.mean().item(), QvalueB=qb.mean().item())
        else:
            q = m.Qaction(obs, act)
            target_q = rew + (1 - ter) * self.gamma * m.Qtarget(nxt)
            q_loss = mse(q, target_q.detach())
            self._step(self.opt_c, m.critic, q_loss)
            p_loss = -m.Qpolicy(obs).mean()
            self._step(self.opt_a, m.actor, p_loss)
            self.sch_a.step()
            self.sch_c.step()
            m.soft_update(self.tau)
            info.update(Qloss=q_loss.item(), Ploss=p_loss.item(), Qvalue=q.mean().item())
        info.update(actor_lr=self.opt_a.param_groups[0]['lr'], critic_lr=self.opt_c.param_groups[0]['lr'])
        return info

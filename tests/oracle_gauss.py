"""Torch-CPU restatement of the reference's PPO update for a Box action space.  TEST INFRASTRUCTURE, in the manner of
oracle/: the reference's arithmetic is torch autograd + torch.distributions + torch.optim, so the same calls are used;
what is restated is the wiring, the loss algebra and the parameter names.

  * SharedActorCritic(Basic_MLP, GaussianActorHead, ValueHead) .. representations/mlp.py:27-57, heads/actor_head.py:45-72,
                                                                  critic_head.py:9-30, actor_critic.py:40-72
  * DiagGaussianDistribution ..................................... modules/distributions.py:165-197
  * PPO-Clip / A2C / PG loss on it ............................... ppo_learner.py:46-60, a2c_learner.py:46-52,
                                                                  pg_learner.py:44-47
Parameter names are the reference's (representation.model.*, actor.mu.*, actor.log_std, critic.values.*), so a state
dict moves between the reference, this restatement and the product model unchanged."""
import torch
import torch.nn as nn
from torch.distributions import Normal

from oracle.learners import PPOLearnerOracle


def _mlp(sizes, act, last_act=None):
    mods = []
    for i in range(len(sizes) - 1):
        mods.append(nn.Linear(sizes[i], sizes[i + 1]))
        if i < len(sizes) - 2:
            mods.append(act())
        elif last_act is not None:
            mods.append(last_act())
    return nn.Sequential(*mods)


class GaussianActorCriticOracle(nn.Module):
    """MLP representation (Linear + activation per hidden size) -> {mu: hidden stack + Linear(->D) + activation_action,
    log_std: Parameter(-1), values: hidden stack + Linear(->1)}.  Returns (mu, log_std, values)."""

    def __init__(self, obs_dim, action_dim, rep_hidden=(64,), actor_hidden=(64,), critic_hidden=(64,),
                 activation=nn.LeakyReLU, activation_action=nn.Tanh):
        super().__init__()
        self.representation = nn.Module()
        self.representation.model = _mlp([obs_dim, *rep_hidden], activation, activation)   # () -> Basic_Identical
        f = rep_hidden[-1] if rep_hidden else obs_dim
        self.actor = nn.Module()
        self.actor.mu = _mlp([f, *actor_hidden, action_dim], activation, activation_action)
        self.actor.log_std = nn.Parameter(-torch.ones(action_dim))
        self.critic = nn.Module()
        self.critic.values = _mlp([f, *critic_hidden, 1], activation)

    def forward(self, obs):
        z = self.representation.model(torch.as_tensor(obs, dtype=torch.float32))
        return self.actor.mu(z), self.actor.log_std, self.critic.values(z).squeeze(-1)


def gauss_dist(mu, log_std):
    """DiagGaussianDistribution.set_param(mu, log_std.exp()) as GaussianActorHead.forward calls it."""
    return Normal(mu, log_std.exp())


def ppo_gauss_terms(mu, log_std, v_pred, act, ret, adv, old_logp, clip_range):
    """ppo_learner.py:46-59 on a DiagGaussianDistribution - returns (a_loss, c_loss, e_loss, ratio)."""
    dist = gauss_dist(mu, log_std)
    log_prob = dist.log_prob(act).sum(-1)
    ratio = (log_prob - old_logp).exp().float()
    surrogate1 = ratio.clamp(1.0 - clip_range, 1.0 + clip_range) * adv
    surrogate2 = adv * ratio
    a_loss = -torch.minimum(surrogate1, surrogate2).mean()
    c_loss = nn.functional.mse_loss(v_pred, ret.detach())
    e_loss = dist.entropy().sum(-1).mean()
    return a_loss, c_loss, e_loss, ratio


def pg_gauss_terms(mu, log_std, act, weight):
    """a2c_learner.py:46-52 / pg_learner.py:44-47 actor term: (-(w * logp).mean(), entropy.mean(), logp)."""
    dist = gauss_dist(mu, log_std)
    log_prob = dist.log_prob(act).sum(-1)
    return -(weight * log_prob).mean(), dist.entropy().sum(-1).mean(), log_prob


class PPOGaussLearnerOracle(PPOLearnerOracle):
    """PPOLearnerOracle's optimiser recipe and info keys, on a model returning (mu, log_std, values)."""

    def update(self, **samples):
        self.iterations += 1
        obs = torch.as_tensor(samples['obs'])
        act = torch.as_tensor(samples['actions'])
        ret = torch.as_tensor(samples['returns'])
        adv = torch.as_tensor(samples['advantages'])
        mu, log_std, v_pred = self.model(obs)
        if self.kind == "ppo":
            old_logp = torch.as_tensor(samples['aux_batch']['old_logp'])
            a_loss, c_loss, e_loss, ratio = ppo_gauss_terms(mu, log_std, v_pred, act, ret, adv, old_logp,
                                                            self.clip_range)
            loss = a_loss - self.ent_coef * e_loss + self.vf_coef * c_loss
        else:
            a_loss, e_loss, log_prob = pg_gauss_terms(mu, log_std, act, adv if self.kind == "a2c" else ret)
            if self.kind == "a2c":
                c_loss = nn.functional.mse_loss(v_pred, ret)
                loss = a_loss - self.ent_coef * e_loss + self.vf_coef * c_loss
            else:
                c_loss = torch.zeros(())
                loss = a_loss - self.ent_coef * e_loss
            ratio = torch.ones_like(log_prob)
        self.optimizer.zero_grad()
        loss.backward()
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(self.model.parameters(), self.grad_clip_norm)
        self.optimizer.step()
        self.scheduler.step()
        lr = self.optimizer.state_dict()['param_groups'][0]['lr']
        cr = ((ratio < 1 - self.clip_range).sum() + (ratio > 1 + self.clip_range).sum()) / ratio.shape[0]
        return {"actor_loss": a_loss.item(), "critic_loss": c_loss.item(), "entropy": e_loss.item(),
                "learning_rate": lr, "predict_value": v_pred.mean().item(), "clip_ratio": cr}

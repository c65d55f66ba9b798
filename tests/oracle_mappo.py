"""Torch-CPU / NumPy oracle of the MAPPO stack, built on ``oracle/`` (its ``mlp`` builder) and independent of the product's
classes; pinned to tests/golden/mappo_update.npz (generated from the unmodified reference).

* ``MAPPOModelOracle``    MultiAgentActorCritic(CategoricalActor, CentralizedStateValueCritic) over Basic_MLP encoders, with
                          the reference's module / parameter names;
* ``MAPPOLearnerOracle``  mappo_learner.py:41-149 with torch autograd, torch.optim.Adam(eps=1e-5), clip_grad_norm_ and
                          the reference's ValueNorm;
* ``MARLOnPolicyBufferOracle`` memory_tools_marl.py:63-270 (store / finish_path / sample) in NumPy."""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.nets import mlp  # noqa: E402
from mappo_refs import finish_path_ref  # noqa: E402


def _box(**children):
    m = nn.Module()
    for k, v in children.items():
        setattr(m, k, v)
    return m


class MAPPOModelOracle(nn.Module):
    """One group 'shared'; ReLU MLPs (no normaliser), orthogonal init as mlp_block does."""

    def __init__(self, obs_dim, n_actions, rep_hidden=(32,), actor_hidden=(32,), critic_hidden=(32,)):
        super().__init__()
        init = nn.init.orthogonal_
        enc = lambda: _box(obs_representation=_box(model=mlp([obs_dim, *rep_hidden], last_act=True, init=init)))
        actor = _box(representation=enc(), actor_head=_box(logits=mlp([rep_hidden[-1], *actor_hidden, n_actions],
                                                                      init=init)))
        critic = _box(representations=nn.ModuleDict({"shared": enc()}),
                      critic_head=_box(values=mlp([rep_hidden[-1], *critic_hidden, 1], init=init)))
        self.actors = nn.ModuleDict({"shared": actor})
        self.critics = nn.ModuleDict({"shared": critic})

    def logits(self, obs):
        a = self.actors["shared"]
        return a.actor_head.logits(a.representation.obs_representation.model(obs))

    def values(self, obs, states=None):
        c = self.critics["shared"]
        x = c.representations["shared"].obs_representation.model(obs)
        if states is not None:
            x = torch.cat([states, x], dim=-1)
        return c.critic_head.values(x).squeeze(-1)


class MARLOnPolicyBufferOracle:
    """Scalar fields [agent, env, T]; finish_path per agent with finish_path_ref (the reference's loop and dtypes)."""

    def __init__(self, n_agents, n_envs, T, use_gae, gamma, lam):
        self.n, self.n_envs, self.T = n_agents, n_envs, T
        self.use_gae, self.gamma, self.lam = use_gae, gamma, lam
        z = lambda: np.zeros((n_agents, n_envs, T), np.float32)
        self.rewards, self.values, self.terminals, self.returns, self.advantages = z(), z(), z(), z(), z()
        self.ptr, self.size, self.start_ids = 0, 0, np.zeros(n_envs, np.int64)

    @property
    def full(self):
        return self.size >= self.T

    def store(self, keys, step):
        for i, k in enumerate(keys):
            self.rewards[i, :, self.ptr] = step['rewards'][k]
            self.values[i, :, self.ptr] = step['values'][k]
            self.terminals[i, :, self.ptr] = step['terminals'][k]
        self.ptr = (self.ptr + 1) % self.T
        self.size = min(self.size + 1, self.T)

    def finish_path(self, i_env, keys, value_next, vn=None):
        """vn: (mean, std) float32 of the ValueNorm state at this call, or None."""
        b, e = int(self.start_ids[i_env]), (self.T if self.full else self.ptr)
        for i, k in enumerate(keys):
            r, a = finish_path_ref(self.rewards[i, i_env, b:e], self.values[i, i_env, b:e],
                                   self.terminals[i, i_env, b:e], value_next[k], self.use_gae, self.gamma, self.lam, vn)
            self.returns[i, i_env, b:e], self.advantages[i, i_env, b:e] = r, a
        self.start_ids[i_env] = self.ptr

    def sample_advantages(self, idx):
        env, step = np.divmod(np.asarray(idx), self.T)
        out = []
        for i in range(self.n):
            a = self.advantages[i, env, step]
            out.append((a - np.mean(a)) / (np.std(a) + 1e-8))
        return np.stack(out)


class ValueNormOracle(nn.Module):
    """value_norm.py:6-75 (input_shape 1)."""

    def __init__(self, beta=0.99999, epsilon=1e-5):
        super().__init__()
        self.beta, self.epsilon = beta, epsilon
        self.running_mean = nn.Parameter(torch.zeros(1), requires_grad=False)
        self.running_mean_sq = nn.Parameter(torch.zeros(1), requires_grad=False)
        self.debiasing_term = nn.Parameter(torch.tensor(0.0), requires_grad=False)

    def running_mean_var(self):
        d = self.debiasing_term.clamp(min=self.epsilon)
        mean, mean_sq = self.running_mean / d, self.running_mean_sq / d
        return mean, (mean_sq - mean ** 2).clamp(min=1e-2)

    @torch.no_grad()
    def update(self, x):
        w = self.beta
        self.running_mean.mul_(w).add_(x.mean(dim=0) * (1.0 - w))
        self.running_mean_sq.mul_(w).add_((x ** 2).mean(dim=0) * (1.0 - w))
        self.debiasing_term.mul_(w).add_(1.0 * (1.0 - w))

    def normalize(self, x):
        mean, var = self.running_mean_var()
        return (x - mean[None]) / torch.sqrt(var)[None]


class MAPPOLearnerOracle:
    def __init__(self, model, cfg):
        self.model, self.cfg = model, cfg
        self.optimizer = torch.optim.Adam(model.parameters(), lr=cfg.learning_rate, eps=1e-5)
        self.vn = ValueNormOracle() if cfg.use_value_norm else None
        self.huber = nn.HuberLoss(reduction="none", delta=cfg.huber_delta)

    def update(self, obs, actions, log_pi_old, adv, values, returns, mask, avail=None, state=None):
        c = self.cfg
        logits = self.model.logits(obs)
        if avail is not None:
            logits[avail == 0] = -1e10
        dist = torch.distributions.Categorical(logits=logits)
        log_pi = dist.log_prob(actions.long())
        ratio = torch.exp(log_pi - log_pi_old)
        s1 = ratio * adv
        s2 = torch.clip(ratio, 1.0 - c.clip_range, 1.0 + c.clip_range) * adv
        actor_loss = -(torch.min(s1, s2) * mask).sum() / mask.sum()
        entropy = dist.entropy()
        entropy_loss = (entropy * mask).sum() / mask.sum()
        v = self.model.values(obs, state)
        target = returns
        if c.use_value_clip:
            v_clipped = values + (v - values).clamp(-c.value_clip_range, c.value_clip_range)
            if self.vn is not None:
                self.vn.update(target.reshape(-1, 1))
                target = self.vn.normalize(target.reshape(-1, 1)).reshape(-1)
            if c.use_huber_loss:
                lv, lvc = self.huber(v, target), self.huber(v_clipped, target)
            else:
                lv, lvc = (v - target) ** 2, (v_clipped - target) ** 2
            critic_loss = (torch.max(lv, lvc) * mask).sum() / mask.sum()
        else:
            if self.vn is not None:
                self.vn.update(target)
                target = self.vn.normalize(target)
            lv = self.huber(v, target) if c.use_huber_loss else (v - target) ** 2
            critic_loss = (lv * mask).sum() / mask.sum()
        loss = actor_loss + c.vf_coef * critic_loss - c.ent_coef * entropy_loss
        self.optimizer.zero_grad()
        loss.backward()
        info = {}
        if c.use_grad_clip:
            info["gradient_norm"] = float(nn.utils.clip_grad_norm_(self.model.parameters(), c.grad_clip_norm))
        self.optimizer.step()
        info.update({"actor_loss": actor_loss.item(), "critic_loss": critic_loss.item(),
                     "entropy": entropy_loss.item(), "predict_value": v.mean().item(), "loss": loss.item()})
        return info

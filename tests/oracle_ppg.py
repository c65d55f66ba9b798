"""Torch autograd oracle of PPG_Learner: ppg_learner.py:38-148 restated, one ``torch.optim.Adam`` over all parameters
(``zero_grad()`` to None, so each phase steps only the parameters its loss reaches) and the LinearLR schedule stepped in
``update_actor`` only; pinned to the reference by tests/golden/ppg_update.npz (test_ppg.py).  Runs on any device, on a model built from this package's classes (their
``forward`` is the reference's); the relabel is ``relabel``, the reference's get_actions + split / merge reduced to the
distribution parameters."""
import torch
import torch.nn.functional as F
from torch.distributions import Categorical, Normal, kl_divergence


class PPGOracle:
    def __init__(self, model, lr, ent_coef, clip_range, kl_beta, use_grad_clip, grad_clip_norm, end_factor_lr_decay,
                 total_iters):
        self.model = model
        self.optimizer = torch.optim.Adam(model.parameters(), lr, eps=1e-5)
        self.scheduler = torch.optim.lr_scheduler.LinearLR(self.optimizer, start_factor=1.0,
                                                           end_factor=end_factor_lr_decay, total_iters=total_iters)
        self.ent_coef, self.clip_range, self.kl_beta = ent_coef, clip_range, kl_beta
        self.use_grad_clip, self.grad_clip_norm = use_grad_clip, grad_clip_norm

    def _step(self, loss):
        self.optimizer.zero_grad()
        loss.backward()
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(self.model.parameters(), self.grad_clip_norm)
        self.optimizer.step()

    def _dist(self, obs):
        return self.model.actor(obs).distributions

    def update_actor(self, obs, act, adv, old_logp):
        a_dist = self._dist(obs)
        log_prob = a_dist.log_prob(act)
        ratio = (log_prob - old_logp).exp().float()
        surrogate1 = ratio.clamp(1.0 - self.clip_range, 1.0 + self.clip_range) * adv
        surrogate2 = adv * ratio
        a_loss = -torch.minimum(surrogate1, surrogate2).mean()
        e_loss = a_dist.entropy().mean()
        self._step(a_loss - self.ent_coef * e_loss)
        self.scheduler.step()
        cr = ((ratio < 1 - self.clip_range).sum() + (ratio > 1 + self.clip_range).sum()) / ratio.shape[0]
        return {"actor-loss": a_loss.item(), "entropy": e_loss.item(),
                "learning_rate": self.optimizer.param_groups[0]['lr'], "clip_ratio": float(cr)}

    def update_critic(self, obs, ret):
        loss = F.mse_loss(self.model.critic(obs).values, ret)
        self._step(loss)
        return {"critic-loss": loss.item()}

    @torch.no_grad()
    def relabel(self, obs):
        """The old distribution's parameters: Categorical logits (log-softmax normalised) or (mu, std [D])."""
        d = self._dist(obs)
        return (d.mu, d.std) if hasattr(d, "mu") else (d.logits,)

    def update_auxiliary_critic(self, obs, ret, old):
        out = self.model(obs)
        a_dist, v = out.distributions, out.values
        aux_v = self.model.aux_critic(obs).values
        if len(old) == 2:
            old_dist = Normal(old[0], old[1].expand_as(old[0]), validate_args=False)
        else:
            old_dist = Categorical(logits=old[0], validate_args=False)
        aux_loss = F.mse_loss(v.detach(), aux_v)
        kl_loss = kl_divergence(a_dist.distribution, old_dist).mean()
        value_loss = F.mse_loss(v, ret)
        loss = aux_loss + self.kl_beta * kl_loss + value_loss
        self._step(loss)
        return {"aux-loss": aux_loss.item(), "kl-loss": kl_loss.item(), "value-loss": value_loss.item(),
                "loss": loss.item()}


def build_fixture_model(kind, device):
    """This package's PhasicActorCritic at a fixture case's shapes (tests/ppg_refs.py FIX_*), weights not yet loaded."""
    import numpy as np
    from copy import deepcopy
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.rl_models import (Basic_MLP, CategoricalActor, GaussianActor, StateValueCritic,
                                             PhasicActorCritic)
    from ppg_refs import FIX_OBS, FIX_HIDDEN, FIX_A, FIX_D
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    rep = Basic_MLP((FIX_OBS,), [FIX_HIDDEN], None, init, act, device)
    if kind == "gauss":
        actor = GaussianActor(rep, [FIX_HIDDEN], Box(-1, 1, (FIX_D,), np.float32), None, init, act, torch.nn.Tanh,
                              device)
    else:
        actor = CategoricalActor(rep, [FIX_HIDDEN], Discrete(FIX_A), None, init, act, device)
    critic = StateValueCritic(deepcopy(rep), [FIX_HIDDEN], None, init, act, device)
    aux_critic = StateValueCritic(deepcopy(rep), [FIX_HIDDEN], None, init, act, device)
    return PhasicActorCritic(actor, critic, aux_critic).to(device)

"""Torch autograd oracle of NPG_Learner: npg_learner.py:26-113 restated with the one correction the reference needs to run
(``distributions`` for ``.distribution``) and with each tensor's F^-1 g in the float64 closed form (tests/npg_refs.py)
instead of the reference's float32 dense inverse.  Two ``torch.optim.Adam`` (eps 1e-5) with LinearLR over
``running_steps``; pinned to the reference by tests/golden/npg_update.npz (test_npg.py).  Runs on any device, on a model
built from this package's classes (their ``forward`` is the reference's)."""
import numpy as np
import torch
import torch.nn.functional as F

from npg_refs import LAM


class NPGOracle:
    def __init__(self, model, lr, use_grad_clip, grad_clip_norm, end_factor_lr_decay, running_steps, horizon_size):
        self.model = model
        self.actor_optimizer = torch.optim.Adam(model.actor.parameters(), lr, eps=1e-5)
        self.critic_optimizer = torch.optim.Adam(model.critic.parameters(), lr, eps=1e-5)
        sched = lambda o: torch.optim.lr_scheduler.LinearLR(o, start_factor=1.0, end_factor=end_factor_lr_decay,
                                                            total_iters=running_steps)
        self.actor_scheduler, self.critic_scheduler = sched(self.actor_optimizer), sched(self.critic_optimizer)
        self.use_grad_clip, self.grad_clip_norm, self.horizon_size = use_grad_clip, grad_clip_norm, horizon_size
        self.natural_grads = None     # the last update's post-clip natural gradient per actor tensor
        self.kappa = None

    def update(self, obs, act, ret, adv):
        out = self.model(obs)
        a_dist, v_pred = out.distributions, out.values
        log_prob = a_dist.log_prob(act)
        a_loss = -(adv * log_prob).mean()
        c_loss = F.mse_loss(v_pred, ret)
        self.critic_optimizer.zero_grad()
        c_loss.backward(retain_graph=True)
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(self.model.critic.parameters(), self.grad_clip_norm)
        self.critic_optimizer.step()
        params = [p for p in self.model.actor.parameters() if p.requires_grad]
        scores = torch.autograd.grad(log_prob.sum(), params, retain_graph=True)
        self.kappa = log_prob.sum().item() / self.horizon_size
        self.actor_optimizer.zero_grad()
        a_loss.backward()
        for p, s in zip(params, scores):
            g64, s64 = p.grad.reshape(-1).double(), s.reshape(-1).double()
            nat = (g64 - s64 * (self.kappa * (s64 @ g64) / (LAM + self.kappa * (s64 @ s64)))) / LAM
            p.grad = nat.to(p.dtype).reshape(p.shape)
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(self.model.actor.parameters(), self.grad_clip_norm)
        self.natural_grads = [p.grad.detach().clone() for p in params]
        self.actor_optimizer.step()
        self.critic_scheduler.step()
        self.actor_scheduler.step()
        lr = self.actor_optimizer.param_groups[0]['lr']
        return {"actor-loss": a_loss.item(), "critic-loss": c_loss.item(), "learning_rate_actor": lr,
                "learning_rate_critic": lr, "predict_value": v_pred.mean().item()}


def build_fixture_model(kind, device):
    """This package's ActorCritic at a fixture case's shapes (tests/npg_refs.py FIX_*), weights not yet loaded."""
    from copy import deepcopy
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.rl_models import Basic_MLP, CategoricalActor, GaussianActor, StateValueCritic, ActorCritic
    from npg_refs import FIX_OBS, FIX_HIDDEN, FIX_A, FIX_D
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    rep = Basic_MLP((FIX_OBS,), [FIX_HIDDEN], None, init, act, device)
    if kind == "gauss":
        actor = GaussianActor(rep, [FIX_HIDDEN], Box(-1, 1, (FIX_D,), np.float32), None, init, act, torch.nn.Tanh,
                              device)
    else:
        actor = CategoricalActor(rep, [FIX_HIDDEN], Discrete(FIX_A), None, init, act, device)
    critic = StateValueCritic(deepcopy(rep), [FIX_HIDDEN], None, init, act, device)
    return ActorCritic(actor, critic).to(device)

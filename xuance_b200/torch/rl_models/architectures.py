"""Model architectures on the hot path (reference: xuance/torch/rl_models/architectures/single_agent/
{actor_critic,deep_q_network}.py, actors/gaussian_actors.py, critics/twin_critics.py).  Same attribute names
so reference checkpoints (``'policy'`` state_dict) load; no DistributedDataParallel wrappers - multi-GPU is ONE
flat-bucket all-reduce issued by the learner (DESIGN.md "Multi-GPU")."""
from copy import deepcopy

import torch
import torch.nn as nn

from ...common.spaces import is_discrete
from .heads import (DuelingQValueHead, QValueHead, SAC_GaussianActorHead, GaussianActorHead, ValueHead,
                    DeterministicActorHead, C51QValueHead, QuantileRegressionQValueHead)
from .outputs import ModelOutput, StochasticActorOutput, TwinCriticOutput, DeterministicActorOutput, CriticOutput


class ActorCritic(nn.Module):
    """actor_critic.py:8-37 (separate actor / critic modules each owning a representation).  ``logits`` / ``mu_log_std``
    and ``forward_raw`` / ``forward_raw_gauss`` give the raw actor outputs (a CategoricalActor's logits, a GaussianActor's
    mu and log_std) and a StateValueCritic's values, the tensors the fused loss and acting kernels consume."""

    def __init__(self, actor, critic, **kwargs):
        super().__init__()
        self.actor, self.critic = actor, critic

    def forward(self, observation, **kwargs):
        a, c = self.actor(observation, **kwargs), self.critic(observation, **kwargs)
        return ModelOutput(distributions=a.distributions, values=c.values, actor_rep_out=a.representations,
                           critic_rep_out=c.representations)

    def act(self, observation, deterministic=False, **kwargs):
        d = self.actor(observation, **kwargs).distributions
        return d.deterministic_sample() if deterministic else d.stochastic_sample()

    def logits(self, observation):
        return self.actor.logits(observation)

    def mu_log_std(self, observation):
        head = self.actor.actor_head
        return head.mu(self.actor.representation(observation).embeddings), head.log_std

    def forward_raw(self, observation):
        """(logits [B, A], values [B])."""
        return self.logits(observation), self.critic.values(observation)

    def forward_raw_gauss(self, observation):
        """(mu [B, D], log_std [D], values [B])."""
        mu, log_std = self.mu_log_std(observation)
        return mu, log_std, self.critic.values(observation)


class SharedActorCritic(nn.Module):
    """actor_critic.py:40-72: representation -> (actor head, critic head)."""

    def __init__(self, representation, actor, critic, **kwargs):
        super().__init__()
        self.representation, self.actor, self.critic = representation, actor, critic

    def forward(self, observation, **kwargs):
        rep_out = self.representation(observation, **kwargs)
        return ModelOutput(distributions=self.actor(rep_out.embeddings, **kwargs),
                           values=self.critic(rep_out.embeddings, **kwargs), rep_out=rep_out)

    def forward_raw(self, observation):
        """(logits, values) without building a torch.distributions object - the fused K4 loss consumes these."""
        z = self.representation(observation).embeddings
        return self.actor.logits(z), self.critic(z)

    def forward_raw_gauss(self, observation):
        """(mu, log_std, values) of a GaussianActorHead without building a torch.distributions object - the fused K4G
        loss and K10G act consume these."""
        z = self.representation(observation).embeddings
        return self.actor.mu(z), self.actor.log_std, self.critic(z)

    def act(self, observation, deterministic=False, **kwargs):
        d = self.actor(self.representation(observation, **kwargs).embeddings, **kwargs)
        return d.deterministic_sample() if deterministic else d.stochastic_sample()


class DeepQNetwork(nn.Module):
    """deep_q_network.py:19-99: eval representation + Q head and their deep-copied targets."""

    q_head_cls = QValueHead

    def __init__(self, representation, hidden_size, action_space=None, normalizer=None, initializer=None,
                 activation=None, device=None, use_distributed_training=False, **kwargs):
        super().__init__()
        if not is_discrete(action_space):
            raise ValueError('action_space must be Discrete')
        self.n_actions = action_space.n
        self.device = device
        self.representation = representation
        self.target_representation = deepcopy(representation)
        self.representation_info_shape = representation.output_shapes
        self.eval_Q_head = self.q_head_cls(feature_dim=self.representation_info_shape['state'][0],
                                           hidden_size=hidden_size, n_actions=self.n_actions, normalizer=normalizer,
                                           initializer=initializer, activation=activation, device=device)
        self.target_Q_head = deepcopy(self.eval_Q_head)
        self.distributed_training = use_distributed_training

    def eval_parameters(self):
        return list(self.representation.parameters()) + list(self.eval_Q_head.parameters())

    def target_parameters(self):
        return list(self.target_representation.parameters()) + list(self.target_Q_head.parameters())

    def forward(self, observation, **kwargs):
        rep = self.representation(observation)
        q = self.eval_Q_head(rep.embeddings)
        return ModelOutput(actions=q.argmax(dim=-1), values=q, rep_out=rep)

    def act(self, observation, deterministic=True, epsilon_greedy=0.0, **kwargs):
        greedy = self(observation).actions
        if deterministic or epsilon_greedy <= 0.0:
            return greedy
        rand = torch.randint(low=0, high=self.n_actions, size=greedy.shape, device=greedy.device)
        mask = torch.rand(greedy.shape, device=greedy.device) < epsilon_greedy
        return torch.where(mask, rand, greedy)

    def target(self, observation, **kwargs):
        rep = self.target_representation(observation)
        return ModelOutput(values=self.target_Q_head(rep.embeddings))

    def copy_target(self):
        for ep, tp in zip(self.representation.parameters(), self.target_representation.parameters()):
            tp.data.copy_(ep)
        for ep, tp in zip(self.eval_Q_head.parameters(), self.target_Q_head.parameters()):
            tp.data.copy_(ep)


class DuelingDeepQNetwork(DeepQNetwork):
    """deep_q_network.py:102-103."""
    q_head_cls = DuelingQValueHead


DIST_MAX_ATOMS, DIST_MAX_ACTIONS = 64, 256     # include/xb200.h K6Z: 2 <= N <= 64 atoms / quantiles, 1 <= A <= 256


class _DistributionalQNetwork(nn.Module):
    """The shared body of C51DeepQNetwork / QRDeepQNetwork: eval representation + distributional head and their
    deep-copied targets.  Greedy actions (and C51's probabilities under no_grad) come from one K6Z ``xb_dist_greedy``
    launch over the head's raw [B, A, N] output; only a forward under autograd builds the reference's softmax in torch,
    for the gradient."""

    head_cls = None
    uses_supports = False

    def __init__(self, representation, hidden_size, action_space, n_atoms, normalizer=None, initializer=None,
                 activation=None, device=None, use_distributed_training=False):
        super().__init__()
        if not is_discrete(action_space):
            raise ValueError('action_space must be Discrete')
        self.n_actions = action_space.n
        if not 2 <= n_atoms <= DIST_MAX_ATOMS:
            raise NotImplementedError("%s supports 2 to %d atoms / quantiles, got %d"
                                      % (type(self).__name__, DIST_MAX_ATOMS, n_atoms))
        if self.n_actions > DIST_MAX_ACTIONS:
            raise NotImplementedError("%s supports at most %d actions, got %d"
                                      % (type(self).__name__, DIST_MAX_ACTIONS, self.n_actions))
        self.device = device
        self.representation = representation
        self.target_representation = deepcopy(representation)
        self.representation_info_shape = representation.output_shapes
        self.eval_Z_head = self.head_cls(feature_dim=self.representation_info_shape['state'][0],
                                         hidden_size=hidden_size, n_actions=self.n_actions, atom_num=n_atoms,
                                         normalizer=normalizer, initializer=initializer, activation=activation,
                                         device=device)
        self.target_Z_head = deepcopy(self.eval_Z_head)
        self.distributed_training = use_distributed_training

    def eval_parameters(self):
        return list(self.representation.parameters()) + list(self.eval_Z_head.parameters())

    def target_parameters(self):
        return list(self.target_representation.parameters()) + list(self.target_Z_head.parameters())

    def forward_raw(self, observation):
        """The eval head's raw [B, A, N] output (C51 logits / QR quantiles), under autograd: the learner's input."""
        return self.eval_Z_head.logits(self.representation(observation).embeddings)

    @torch.no_grad()
    def target_raw(self, observation):
        return self.target_Z_head.logits(self.target_representation(observation).embeddings)

    def greedy(self, z, with_probs=False):
        """One ``xb_dist_greedy`` launch over raw [B, A, N] -> (actions int64 [B], C51 probabilities or None)."""
        from ... import _lib
        z = z.detach().to(torch.float32).contiguous()
        B, A, N = z.shape
        actions = torch.empty(B, dtype=torch.int64, device=z.device)
        probs = torch.empty_like(z) if with_probs else None
        sup = self.supports if self.uses_supports else None
        _lib.call("xb_dist_greedy", _lib.ptr(z), _lib.ptr(sup), B, A, N, _lib.ptr(actions), None, _lib.ptr(probs))
        return actions, probs

    def _output(self, z, rep=None):
        if torch.is_grad_enabled() and z.requires_grad:
            actions, _ = self.greedy(z)
            values = torch.softmax(z, dim=-1) if self.uses_supports else z
        else:
            actions, probs = self.greedy(z, with_probs=self.uses_supports)
            values = probs if self.uses_supports else z
        return ModelOutput(actions=actions, values=values, rep_out=rep)

    def forward(self, observation, **kwargs):
        rep = self.representation(observation)
        return self._output(self.eval_Z_head.logits(rep.embeddings), rep)

    @torch.no_grad()
    def greedy_actions(self, observation):
        """The eval network's greedy actions alone: one xb_dist_greedy launch that writes no probabilities (acting)."""
        return self.greedy(self.eval_Z_head.logits(self.representation(observation).embeddings))[0]

    def act(self, observation, deterministic=True, epsilon_greedy=0.0, **kwargs):
        greedy = self.greedy_actions(observation)
        if deterministic or epsilon_greedy <= 0.0:
            return greedy
        rand = torch.randint(low=0, high=self.n_actions, size=greedy.shape, device=greedy.device)
        mask = torch.rand(greedy.shape, device=greedy.device) < epsilon_greedy
        return torch.where(mask, rand, greedy)

    def target(self, observation, **kwargs):
        rep = self.target_representation(observation)
        out = self._output(self.target_Z_head.logits(rep.embeddings))
        return ModelOutput(actions=out.actions, values=out.values)

    def copy_target(self):
        for ep, tp in zip(self.representation.parameters(), self.target_representation.parameters()):
            tp.data.copy_(ep)
        for ep, tp in zip(self.eval_Z_head.parameters(), self.target_Z_head.parameters()):
            tp.data.copy_(ep)


class C51DeepQNetwork(_DistributionalQNetwork):
    """deep_q_network.py:146-238.  ``supports`` is a registered, frozen Parameter filled by torch.linspace on the CPU (the
    values a CPU-built reference model holds and saves in its state_dict; DESIGN section 4)."""

    head_cls = C51QValueHead
    uses_supports = True

    def __init__(self, representation, hidden_size, action_space, atom_num, v_min, v_max, normalizer=None,
                 initializer=None, activation=None, device=None, use_distributed_training=False, **kwargs):
        super().__init__(representation, hidden_size, action_space, atom_num, normalizer, initializer, activation,
                         device, use_distributed_training)
        self.atom_num, self.v_min, self.v_max = atom_num, v_min, v_max
        self.supports = nn.Parameter(torch.linspace(v_min, v_max, atom_num).to(device), requires_grad=False)
        self.delta_z = (v_max - v_min) / (atom_num - 1)


class QRDeepQNetwork(_DistributionalQNetwork):
    """deep_q_network.py:241-325."""

    head_cls = QuantileRegressionQValueHead

    def __init__(self, representation, hidden_size, action_space, quantile_num, normalizer=None, initializer=None,
                 activation=None, device=None, use_distributed_training=False, **kwargs):
        super().__init__(representation, hidden_size, action_space, quantile_num, normalizer, initializer, activation,
                         device, use_distributed_training)
        self.quantile_num = quantile_num


class GaussianActor(nn.Module):
    """actors/gaussian_actors.py:10-52."""

    actor_head_cls = GaussianActorHead

    def __init__(self, representation, actor_hidden_size, action_space=None, normalizer=None, initializer=None,
                 activation=None, activation_action=None, device=None, **kwargs):
        super().__init__()
        self.action_space = action_space
        self.action_dim = action_space.shape[0]
        self.representation = representation
        self.representation_info_shape = representation.output_shapes
        self.actor_head = self.actor_head_cls(feature_dim=self.representation_info_shape['state'][0],
                                              hidden_size=actor_hidden_size, action_dim=self.action_dim,
                                              normalizer=normalizer, initializer=initializer, activation=activation,
                                              activation_action=activation_action, device=device)

    def forward(self, observation, avail_actions=None, **kwargs):
        rep_out = self.representation(observation, **kwargs)
        return StochasticActorOutput(representations=rep_out,
                                     distributions=self.actor_head(rep_out.embeddings, **kwargs))


class SAC_GaussianActor(GaussianActor):
    actor_head_cls = SAC_GaussianActorHead


class TwinActionValueCritic(nn.Module):
    """critics/twin_critics.py:11-62: two (representation, ValueHead) towers over concat(features, action)."""

    def __init__(self, representation, action_space, critic_hidden_size, normalizer=None, initializer=None,
                 activation=None, device=None, **kwargs):
        super().__init__()
        self.action_space = action_space
        self.action_dim = action_space.shape[-1]
        self.representation_1 = representation
        self.representation_2 = deepcopy(representation)
        self.representation_info_shape = representation.output_shapes
        self.feature_dim = self.representation_info_shape['state'][0] + self.action_dim
        kw = dict(feature_dim=self.feature_dim, hidden_size=critic_hidden_size, normalizer=normalizer,
                  initializer=initializer, activation=activation, device=device)
        self.critic_head_1 = ValueHead(**kw)
        self.critic_head_2 = ValueHead(**kw)

    def forward(self, observation, actions, **kwargs):
        r1, r2 = self.representation_1(observation), self.representation_2(observation)
        return TwinCriticOutput(
            representations_1=r1, representations_2=r2,
            values_1=self.critic_head_1(torch.concat([r1.embeddings, actions], dim=-1)),
            values_2=self.critic_head_2(torch.concat([r2.embeddings, actions], dim=-1)))


class SoftActorCritic(ActorCritic):
    """actor_critic.py:107-159."""

    def __init__(self, actor, critic, **kwargs):
        super().__init__(actor, critic, **kwargs)
        self.target_critic = deepcopy(critic)

    def forward(self, observation, **kwargs):
        a = self.actor(observation, **kwargs)
        c = self.critic(observation, a.actions, **kwargs)
        return ModelOutput(distributions=a.distributions, values=c, actor_rep_out=a.representations)

    def act(self, observation, deterministic=False, **kwargs):
        d = self.actor(observation, **kwargs).distributions
        return d.activated_deterministic_sample() if deterministic else d.activated_rsample()

    def Qpolicy(self, observation, noise=None):
        d = self.actor(observation).distributions
        act_sample, log_prob = d.activated_rsample_and_logprob(noise)
        v1, v2 = self.Qaction(observation, act_sample)
        return log_prob, v1, v2

    def Qtarget(self, observation, noise=None):
        d = self.actor(observation).distributions
        act_sample, log_prob = d.activated_rsample_and_logprob(noise)
        out = self.target_critic(observation, act_sample)
        return log_prob, torch.min(out.values_1, out.values_2)

    def Qaction(self, observation, action):
        out = self.critic(observation, action)
        return out.values_1, out.values_2

    def soft_update(self, tau=0.005):
        for ep, tp in zip(self.critic.parameters(), self.target_critic.parameters()):
            tp.data.mul_(1 - tau)
            tp.data.add_(tau * ep.data)


class TwinDiscreteActionValueCritic(nn.Module):
    """critics/twin_critics.py:65-117: two (representation, QValueHead) towers, each giving Q(s, .) over the A actions."""

    def __init__(self, representation, action_space, critic_hidden_size, normalizer=None, initializer=None,
                 activation=None, device=None, **kwargs):
        super().__init__()
        if not is_discrete(action_space):
            raise ValueError('action_space must be Discrete')
        self.action_space = action_space
        self.n_actions = action_space.n
        self.representation_1 = representation
        self.representation_2 = deepcopy(representation)
        self.representation_info_shape = representation.output_shapes
        self.feature_dim = self.representation_info_shape['state'][0]
        kw = dict(feature_dim=self.feature_dim, hidden_size=critic_hidden_size, n_actions=self.n_actions,
                  normalizer=normalizer, initializer=initializer, activation=activation, device=device)
        self.critic_head_1 = QValueHead(**kw)
        self.critic_head_2 = QValueHead(**kw)

    def forward(self, observation, **kwargs):
        r1, r2 = self.representation_1(observation), self.representation_2(observation)
        return TwinCriticOutput(representations_1=r1, representations_2=r2,
                                values_1=self.critic_head_1(r1.embeddings), values_2=self.critic_head_2(r2.embeddings))


class SoftActorCriticDiscrete(SoftActorCritic):
    """actor_critic.py:162-214 over a CategoricalActor.  Qpolicy / Qtarget / Qaction return the raw logits and [B, A] Q
    matrices: the probability and log rules (p = softmax, log(p + 1e-8*[p == 0])) and the losses run in the K8D kernels,
    and the agent samples with K10."""

    def forward(self, observation, **kwargs):
        """The reference returns the actor's distribution and the critic's output; here the raw logits stand in for the
        distribution (``actor_rep_out``)."""
        return ModelOutput(values=self.critic(observation), actor_rep_out=self.actor.logits(observation))

    def act(self, observation, deterministic=False, **kwargs):
        """K10 ``xb_categorical_act`` on the actor's logits: inverse-CDF sampling of uniforms, or the first argmax when
        ``deterministic``.  Returns int32 actions [N]."""
        from ... import _lib
        logits = self.actor.logits(observation).contiguous()
        N, A = logits.shape
        u = None if deterministic else torch.rand(N, device=logits.device)
        actions = torch.empty(N, dtype=torch.int32, device=logits.device)
        _lib.call("xb_categorical_act", _lib.ptr(logits), _lib.ptr(u), None, N, A, None, _lib.ptr(actions), None, None)
        return actions

    def Qpolicy(self, observation):
        q1, q2 = self.Qaction(observation)
        return self.actor.logits(observation), q1, q2

    def Qtarget(self, observation):
        out = self.target_critic(observation)
        return self.actor.logits(observation), out.values_1, out.values_2

    def Qaction(self, observation, *args, **kwargs):
        out = self.critic(observation)
        return out.values_1, out.values_2


class DeterministicActor(nn.Module):
    """actors/deterministic_actors.py:10-52.  ``action_low`` / ``action_high`` are float32 device tensors (plain
    attributes, as in the reference, so they are not part of the state_dict)."""

    actor_head_cls = DeterministicActorHead

    def __init__(self, representation, actor_hidden_size, action_space=None, normalizer=None, initializer=None,
                 activation=None, activation_action=None, device=None, **kwargs):
        super().__init__()
        if is_discrete(action_space) or not hasattr(action_space, "low"):
            raise ValueError('action_space must be Box')
        self.action_space = action_space
        self.action_dim = action_space.shape[0]
        self.action_low = torch.as_tensor(action_space.low, dtype=torch.float32, device=device)
        self.action_high = torch.as_tensor(action_space.high, dtype=torch.float32, device=device)
        self.representation = representation
        self.representation_info_shape = representation.output_shapes
        self.actor_head = self.actor_head_cls(feature_dim=self.representation_info_shape['state'][0],
                                              hidden_size=actor_hidden_size, action_dim=self.action_dim,
                                              normalizer=normalizer, initializer=initializer, activation=activation,
                                              activation_action=activation_action, device=device)

    def forward(self, observation, **kwargs):
        rep_out = self.representation(observation, **kwargs)
        return DeterministicActorOutput(representations=rep_out, actions=self.actor_head(rep_out.embeddings, **kwargs))


class ActionValueCritic(nn.Module):
    """critics/base_critics.py:47-88: Q(s, a) = ValueHead(concat(features, action))."""

    def __init__(self, representation, action_space, critic_hidden_size, normalizer=None, initializer=None,
                 activation=None, device=None, **kwargs):
        super().__init__()
        if is_discrete(action_space) or not hasattr(action_space, "low"):
            raise ValueError('action_space must be Box.')
        self.action_space = action_space
        self.action_dim = action_space.shape[-1]
        self.representation = representation
        self.representation_info_shape = representation.output_shapes
        self.critic_head = ValueHead(feature_dim=self.representation_info_shape['state'][0] + self.action_dim,
                                     hidden_size=critic_hidden_size, normalizer=normalizer, initializer=initializer,
                                     activation=activation, device=device)

    def forward(self, observations, actions, **kwargs):
        rep_out = self.representation(observations, **kwargs)
        return CriticOutput(representations=rep_out,
                            values=self.critic_head(torch.concat([rep_out.embeddings, actions], dim=-1)))


class DeterministicActorCritic(nn.Module):
    """actor_critic.py:217-261: actor, critic and their deep-copied targets.  ``Qtarget_pair`` / ``Qpolicy_pair`` give
    the learner the raw critic outputs ((q, None) for one critic); the losses run in the K8T kernels."""

    def __init__(self, actor, critic, **kwargs):
        super().__init__()
        self.actor, self.critic = actor, critic
        self.target_actor = deepcopy(actor)
        self.target_critic = deepcopy(critic)

    def forward(self, observations, **kwargs):
        a = self.actor(observations, **kwargs)
        c = self.critic(observations, a.actions, **kwargs)
        return ModelOutput(actions=a.actions, values=c.values, actor_rep_out=a.representations,
                           critic_rep_out=c.representations)

    def act(self, observation, **kwargs):
        return self.actor(observation, **kwargs).actions

    def Qtarget_pair(self, observation, noise=None):
        return self.target_critic(observation, self.target_actor(observation).actions).values, None

    def Qpolicy_pair(self, observation):
        return self.critic(observation, self.actor(observation).actions).values, None

    def Qtarget(self, observation):
        return self.Qtarget_pair(observation)[0]

    def Qaction(self, observations, actions):
        return self.critic(observations, actions).values

    def Qpolicy(self, observation):
        return self.Qpolicy_pair(observation)[0]

    def soft_update(self, tau=0.005):
        for src, dst in ((self.actor, self.target_actor), (self.critic, self.target_critic)):
            for ep, tp in zip(src.parameters(), dst.parameters()):
                tp.data.mul_(1 - tau)
                tp.data.add_(tau * ep.data)


class TwinDelayedActorCritic(DeterministicActorCritic):
    """actor_critic.py:264-319 over a TwinActionValueCritic.  Target-policy smoothing runs in K8T
    ``xb_perturb_actions``: clamp(a' + clip(noise*target_policy_noise, +-target_noise_clip), action_low, action_high)
    with ``noise`` a standard normal [B, action_dim] tensor (drawn with torch.randn_like when not given)."""

    def __init__(self, actor, critic, target_policy_noise=0.2, target_noise_clip=0.5, **kwargs):
        super().__init__(actor, critic, **kwargs)
        self.target_policy_noise = target_policy_noise
        self.target_noise_clip = target_noise_clip

    def forward(self, observation, **kwargs):
        a = self.actor(observation)
        return ModelOutput(actions=a.actions, actor_rep_out=a.representations)

    def smoothed_target_actions(self, observation, noise=None):
        from ... import _lib
        ta = self.target_actor(observation).actions.contiguous()
        noise = torch.randn_like(ta) if noise is None else noise.to(torch.float32).contiguous()
        out = torch.empty_like(ta)
        B, D = ta.shape
        _lib.call("xb_perturb_actions", _lib.ptr(ta), _lib.ptr(noise), B, D, float(self.target_policy_noise),
                  float(self.target_noise_clip), _lib.ptr(self.actor.action_low), _lib.ptr(self.actor.action_high),
                  _lib.ptr(out))
        return out

    def Qtarget_pair(self, observation, noise=None):
        out = self.target_critic(observation, self.smoothed_target_actions(observation, noise))
        return out.values_1, out.values_2

    def Qpolicy_pair(self, observation):
        out = self.critic(observation, self.actor(observation).actions)
        return out.values_1, out.values_2

    def Qtarget(self, observation, noise=None):
        return torch.minimum(*self.Qtarget_pair(observation, noise))

    def Qaction(self, observations, actions):
        out = self.critic(observations, actions)
        return out.values_1, out.values_2

    def Qpolicy(self, observation):
        q1, q2 = self.Qpolicy_pair(observation)
        return (q1 + q2) / 2.0


class StateValueCritic(nn.Module):
    """critics/base_critics.py:11-43: V(s) = ValueHead(representation(s))."""

    def __init__(self, representation, critic_hidden_size, normalizer=None, initializer=None, activation=None,
                 device=None, **kwargs):
        super().__init__()
        self.representation = representation
        self.representation_info_shape = representation.output_shapes
        self.critic_head = ValueHead(feature_dim=self.representation_info_shape['state'][0],
                                     hidden_size=critic_hidden_size, normalizer=normalizer, initializer=initializer,
                                     activation=activation, device=device)

    def values(self, observation):
        """The [B] values alone."""
        return self.critic_head(self.representation(observation).embeddings)

    def forward(self, observation, **kwargs):
        rep_out = self.representation(observation, **kwargs)
        return CriticOutput(representations=rep_out, values=self.critic_head(rep_out.embeddings))


class PhasicActorCritic(ActorCritic):
    """actor_critic.py:75-104: an actor (CategoricalActor or GaussianActor) and two StateValueCritics, each with its own
    representation, sharing no parameter.  ``forward`` returns the actor's distribution and ``critic``'s values.
    Parameters are registered actor, critic, aux_critic: ``parameters()`` lists the three groups in that order, the
    layout the PPG learner's per-group Adam steps by range.  The raw-output methods are ActorCritic's."""

    def __init__(self, actor, critic, aux_critic, **kwargs):
        super().__init__(actor, critic, **kwargs)
        self.aux_critic = aux_critic

    def aux_values(self, observation):
        """``aux_critic``'s [B] values."""
        return self.aux_critic.values(observation)

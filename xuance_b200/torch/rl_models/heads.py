"""Network heads (reference: xuance/torch/rl_models/heads/{actor_head,critic_head,q_head}.py) - same module /
parameter names (``logits``, ``values``, ``q_value``, ``output``/``out_mu``/``out_log_std``)."""
import torch
import torch.nn as nn

from .layers import mlp_block
from .distributions import CategoricalDistribution, DiagGaussianDistribution, ActivatedDiagGaussianDistribution


def _stack(feature_dim, hidden_size, normalizer, activation, initializer, device):
    layers, shape = [], (feature_dim,)
    for h in hidden_size:
        mlp, shape = mlp_block(shape[0], h, normalizer, activation, initializer, device)
        layers.extend(mlp)
    return layers, shape


class CategoricalActorHead(nn.Module):
    """actor_head.py:14-42."""

    def __init__(self, feature_dim, hidden_size, action_dim, normalizer=None, initializer=None, activation=None,
                 device=None, **kwargs):
        super().__init__()
        layers, shape = _stack(feature_dim, hidden_size, normalizer, activation, initializer, device)
        layers.extend(mlp_block(shape[0], action_dim, None, None, initializer, device)[0])
        self.logits = nn.Sequential(*layers)
        self.policy_distribution = CategoricalDistribution(action_dim=action_dim)

    def forward(self, features, avail_actions=None, **kwargs):
        logits = self.logits(features)
        if avail_actions is not None:
            logits[avail_actions == 0] = -1e10
        self.policy_distribution.set_param(logits=logits)
        return self.policy_distribution


class GaussianActorHead(nn.Module):
    """actor_head.py:45-72."""

    def __init__(self, feature_dim, hidden_size, action_dim, normalizer=None, initializer=None, activation=None,
                 activation_action=None, device=None, **kwargs):
        super().__init__()
        layers, shape = _stack(feature_dim, hidden_size, normalizer, activation, initializer, device)
        layers.extend(mlp_block(shape[0], action_dim, None, activation_action, initializer, device)[0])
        self.mu = nn.Sequential(*layers)
        self.log_std = nn.Parameter(-torch.ones((action_dim,), device=device))
        self.policy_distribution = DiagGaussianDistribution(action_dim)

    def forward(self, features, avail_actions=None, **kwargs):
        self.policy_distribution.set_param(self.mu(features), self.log_std.exp())
        return self.policy_distribution


class SAC_GaussianActorHead(nn.Module):
    """actor_head.py:75-105: shared trunk, separate mu / log_std linears, log_std clamped to [-20, 2]."""

    def __init__(self, feature_dim, hidden_size, action_dim, normalizer=None, initializer=None, activation=None,
                 activation_action=None, device=None, **kwargs):
        super().__init__()
        layers, _ = _stack(feature_dim, hidden_size, normalizer, activation, initializer, device)
        self.output = nn.Sequential(*layers)
        self.out_mu = nn.Linear(hidden_size[-1], action_dim, device=device)
        self.out_log_std = nn.Linear(hidden_size[-1], action_dim, device=device)
        self.policy_distribution = ActivatedDiagGaussianDistribution(action_dim, activation_action, device)

    def forward(self, features, avail_actions=None, **kwargs):
        output = self.output(features)
        mu = self.out_mu(output)
        log_std = torch.clamp(self.out_log_std(output), -20, 2)
        self.policy_distribution.set_param(mu, log_std.exp())
        return self.policy_distribution


class DeterministicActorHead(nn.Module):
    """actor_head.py:108-135: hidden layers, then Linear(action_dim) + activation_action (tanh in every shipped config)."""

    def __init__(self, feature_dim, hidden_size, action_dim, normalizer=None, initializer=None, activation=None,
                 activation_action=None, device=None, **kwargs):
        super().__init__()
        layers, shape = _stack(feature_dim, hidden_size, normalizer, activation, initializer, device)
        layers.extend(mlp_block(shape[0], action_dim, None, activation_action, initializer, device)[0])
        self.model = nn.Sequential(*layers)

    def forward(self, features, avail_actions=None, **kwargs):
        actions = self.model(features)
        if avail_actions is not None:
            actions[avail_actions == 0] = 0
        return actions


class ValueHead(nn.Module):
    """critic_head.py:9-30."""

    def __init__(self, feature_dim, hidden_size, normalizer=None, initializer=None, activation=None, device=None,
                 **kwargs):
        super().__init__()
        layers, shape = _stack(feature_dim, hidden_size, normalizer, activation, initializer, device)
        layers.extend(mlp_block(shape[0], 1, None, None, initializer, device)[0])
        self.values = nn.Sequential(*layers)

    def forward(self, features, **kwargs):
        return self.values(features).squeeze(-1)


class QValueHead(nn.Module):
    """q_head.py:11-39."""

    def __init__(self, feature_dim, hidden_size, n_actions, normalizer=None, initializer=None, activation=None,
                 device=None, **kwargs):
        super().__init__()
        self.feature_dim, self.n_actions = feature_dim, n_actions
        layers, shape = _stack(feature_dim, hidden_size, normalizer, activation, initializer, device)
        layers.extend(mlp_block(shape[0], n_actions, None, None, initializer, device)[0])
        self.q_value = nn.Sequential(*layers)

    def forward(self, features, avail_actions=None, **kwargs):
        q_values = self.q_value(features)
        if avail_actions is not None:
            q_values[avail_actions == 0] = -1e10
        return q_values


class DuelingQValueHead(nn.Module):
    """q_head.py:42-80: Q = V + (A - mean(A)); both streams use hidden sizes h // 2.  (The reference hands the NORMALISER
    where the last layers' initialiser belongs, so those two layers keep torch's default initialisation - kept.)"""

    def __init__(self, feature_dim, hidden_size, n_actions, normalizer=None, initializer=None, activation=None,
                 device=None, **kwargs):
        super().__init__()
        self.feature_dim, self.n_actions = feature_dim, n_actions
        half = [h // 2 for h in hidden_size]
        v_layers, shape = _stack(feature_dim, half, normalizer, activation, initializer, device)
        v_layers.extend(mlp_block(shape[0], 1, None, None, None, device)[0])
        self.v_model = nn.Sequential(*v_layers)
        a_layers, shape = _stack(feature_dim, half, normalizer, activation, initializer, device)
        a_layers.extend(mlp_block(shape[0], n_actions, None, None, None, device)[0])
        self.a_model = nn.Sequential(*a_layers)

    def forward(self, features, avail_actions=None, **kwargs):
        values, advantages = self.v_model(features), self.a_model(features)
        q_values = values + (advantages - advantages.mean(dim=-1).unsqueeze(dim=-1))
        if avail_actions is not None:
            q_values[avail_actions == 0] = -1e10
        return q_values


class C51QValueHead(nn.Module):
    """q_head.py:83-114: hidden layers, then Linear(n_actions * atom_num).  ``logits`` is the raw [B, A, N] view the
    K6Z kernels consume; ``forward`` is the reference's softmax over atoms (autograd path)."""

    def __init__(self, feature_dim, hidden_size, n_actions, atom_num, normalizer=None, initializer=None,
                 activation=None, device=None, **kwargs):
        super().__init__()
        self.feature_dim, self.n_actions, self.atom_num = feature_dim, n_actions, atom_num
        layers, shape = _stack(feature_dim, hidden_size, normalizer, activation, initializer, device)
        layers.extend(mlp_block(shape[0], n_actions * atom_num, None, None, initializer, device)[0])
        self.model = nn.Sequential(*layers)

    def logits(self, features):
        return self.model(features).view(-1, self.n_actions, self.atom_num)

    def forward(self, features, avail_actions=None, **kwargs):
        if avail_actions is not None:
            raise NotImplementedError("action masks are not supported by the distributional Q heads")
        return torch.softmax(self.logits(features), dim=-1)


class QuantileRegressionQValueHead(C51QValueHead):
    """q_head.py:117-123: the same layers; the output is the [B, A, N] quantiles themselves."""

    def forward(self, features, avail_actions=None, **kwargs):
        if avail_actions is not None:
            raise NotImplementedError("action masks are not supported by the distributional Q heads")
        return self.logits(features)

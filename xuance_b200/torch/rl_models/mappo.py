"""MAPPO model pieces - mirrors of CategoricalActor (xuance/torch/rl_models/actors/categorical_actors.py:10-48),
CentralizedStateValueCritic (critics/centralized_critics.py:13-93) and MultiAgentActorCritic
(architectures/multi_agent/actor_critic.py:173-...) for one parameter-sharing group of feed-forward agents.  Module /
parameter names follow the reference (``actors.<group>.representation.obs_representation.*``,
``actors.<group>.actor_head.logits.*``, ``critics.<group>.representations.<group>.obs_representation.*``,
``critics.<group>.critic_head.values.*``), so its ``state_dict`` loads unchanged.

The models work on PACKED rows: one row per (sample, agent), the layout the buffer gathers.  ``logits`` are the raw
actor outputs; the action mask is applied by the consumer (the fused loss kernel, or the acting path)."""
import torch
import torch.nn as nn

from .heads import CategoricalActorHead, ValueHead


class CategoricalActor(nn.Module):
    def __init__(self, representation, actor_hidden_size, action_space=None, normalizer=None, initializer=None,
                 activation=None, device=None, **kwargs):
        super().__init__()
        if not hasattr(action_space, "n"):
            raise ValueError('action_space must be Discrete')
        self.action_dim = action_space.n
        self.representation = representation
        self.representation_info_shape = representation.output_shapes
        self.actor_head = CategoricalActorHead(feature_dim=self.representation_info_shape['state'][0],
                                               hidden_size=actor_hidden_size, action_dim=self.action_dim,
                                               normalizer=normalizer, initializer=initializer, activation=activation,
                                               device=device)

    def logits(self, observations):
        return self.actor_head.logits(self.representation(observations).embeddings)


class CentralizedStateValueCritic(nn.Module):
    """V(s, o^i): each agent's value from its own observation embedding (and the global state when given), as the
    reference stacks the per-agent embeddings and applies the head row by row."""

    def __init__(self, grouping, representations, state_space, critic_hidden_size, normalizer=None, initializer=None,
                 activation=None, use_rnn=False, device=None, **kwargs):
        super().__init__()
        self.grouping, self.group_keys = grouping, grouping.group_keys
        self.state_dim = 0 if state_space is None else int(state_space.shape[0])
        self.representations = representations
        emb = sum(representations[k].output_shapes['state'][0] for k in self.group_keys)
        self.critic_head = ValueHead(feature_dim=self.state_dim + emb, hidden_size=critic_hidden_size,
                                     normalizer=normalizer, initializer=initializer, activation=activation,
                                     device=device)

    def values(self, observations, states=None):
        x = self.representations[self.group_keys[0]](observations).embeddings
        if states is not None:
            x = torch.cat([states, x], dim=-1)
        return self.critic_head(x)


class MultiAgentActorCritic(nn.Module):
    def __init__(self, grouping, actors, critics, use_rnn=False, device=None, **kwargs):
        super().__init__()
        if use_rnn:
            raise NotImplementedError("recurrent MAPPO (use_rnn=True, MARL_OnPolicyBuffer_RNN) is not supported")
        self.grouping, self.group_keys = grouping, grouping.group_keys
        self.actors, self.critics = actors, critics

    def logits(self, observations, group=None):
        return self.actors[group or self.group_keys[0]].logits(observations)

    def values(self, observations, states=None, group=None):
        return self.critics[group or self.group_keys[0]].values(observations, states)

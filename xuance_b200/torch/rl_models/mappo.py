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
from .outputs import StochasticActorOutput


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

    def forward(self, observation, avail_actions=None, **kwargs):
        """categorical_actors.py:38-48: the representation's output and the head's CategoricalDistribution."""
        rep_out = self.representation(observation, **kwargs)
        return StochasticActorOutput(representations=rep_out,
                                     distributions=self.actor_head(rep_out.embeddings, avail_actions=avail_actions))

    def logits(self, observations, rnn_states=None, return_states=False):
        """Recurrent representations take [S, T, obs] (or [S, obs] for one step) and the state [1, S, H]."""
        rep = self.representation(observations, rnn_hidden=rnn_states)
        out = self.actor_head.logits(rep.embeddings)
        return (out, rep.rnn_states) if return_states else out


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

    def values(self, observations, states=None, rnn_states=None, return_states=False):
        rep = self.representations[self.group_keys[0]](observations, rnn_hidden=rnn_states)
        x = rep.embeddings
        if states is not None:
            x = torch.cat([states, x], dim=-1)
        out = self.critic_head(x)
        return (out, rep.rnn_states) if return_states else out


class MultiAgentActorCritic(nn.Module):
    def __init__(self, grouping, actors, critics, use_rnn=False, device=None, **kwargs):
        super().__init__()
        self.grouping, self.group_keys = grouping, grouping.group_keys
        self.actors, self.critics = actors, critics
        self.use_rnn = use_rnn

    def logits(self, observations, group=None, rnn_states=None, return_states=False):
        return self.actors[group or self.group_keys[0]].logits(observations, rnn_states, return_states)

    def values(self, observations, states=None, group=None, rnn_states=None, return_states=False):
        return self.critics[group or self.group_keys[0]].values(observations, states, rnn_states, return_states)

    # ---- recurrent states (actor_critic.py init_rnn_states / init_rnn_states_item): rows are (env, agent) pairs
    def _rnn(self, part):
        g = self.group_keys[0]
        return (self.actors[g].representation if part == "actor" else self.critics[g].representations[g]).obs_representation

    def init_rnn_states(self, n_rows):
        """Zero actor and critic hidden states [1, n_rows, H] on the device."""
        return self._rnn("actor").init_rnn_states(n_rows), self._rnn("critic").init_rnn_states(n_rows)

    def init_rnn_states_item(self, rows, rnn_states_actor, rnn_states_critic=None):
        """Zero the rows of a finished env in place, on the device."""
        rnn_states_actor[:, rows] = 0.0
        if rnn_states_critic is not None:
            rnn_states_critic[:, rows] = 0.0
        return rnn_states_actor, rnn_states_critic

"""COMA model pieces - mirrors of CounterfactualCentralizedCritic (xuance/torch/rl_models/critics/centralized_critics.py:
202-293) and CounterfactualMultiAgentActorCritic (architectures/multi_agent/actor_critic.py:244-346) for one
parameter-sharing group.  Module / parameter names follow the reference (``actors.<group>.representation.obs_representation.*``,
``actors.<group>.actor_head.*``, ``critics.representations.<group>.obs_representation.*``, ``critics.critic_head.q_value.*``
and the same under ``target_critics.``), so its ``state_dict`` loads unchanged.

Rows are agent steps in the episode buffer's (b, i, t) order, r = (b*n + i)*T + t.  The critic input of a row is
[state(b, t) | critic features(b, i, t) | joint one-hot of the agents' actions at (b, t), agent i's block zeroed],
assembled by K4C ``xb_coma_critic_input`` in one launch.  ``logits`` are the raw actor outputs: the action mask and the
epsilon mix are applied by the consumers (K4C's loss and acting kernels)."""
import copy

import torch
import torch.nn as nn

from ... import _lib
from .heads import QValueHead


class CriticInput(torch.autograd.Function):
    """K4C xb_coma_critic_input.  state [B, T, S], feat [R, F], actions [B, n, T] (float32 integers) -> [R, S+F+n*A].
    The backward is the feature slice of the output gradient; state and actions take no gradient."""

    @staticmethod
    def forward(ctx, state, feat, actions, n, A):
        B, T, S = state.shape
        R, F = feat.shape
        out = torch.empty((R, S + F + n * A), dtype=torch.float32, device=feat.device)
        _lib.call("xb_coma_critic_input", _lib.ptr(state), _lib.ptr(feat), _lib.ptr(actions), B, n, T, S, F, A,
                  _lib.ptr(out))
        ctx.S, ctx.F = S, F
        return out

    @staticmethod
    def backward(ctx, g):
        return None, g[:, ctx.S:ctx.S + ctx.F], None, None, None


def critic_input(state, feat, actions, n, A):
    """The COMA critic input rows (see CriticInput); inputs are made contiguous float32."""
    f = lambda x: x.to(torch.float32).contiguous()
    return CriticInput.apply(f(state), f(feat), f(actions), n, A)


class CounterfactualCentralizedCritic(nn.Module):
    """Q(s, o^i, a^{-i}, .) for every action of agent i: the critic encoder (``representations[group]``), then
    K4C's input assembly, then ``critic_head`` (QValueHead over S + H + n*A inputs, A outputs)."""

    def __init__(self, grouping, representations, state_space, action_space, critic_hidden_size, normalizer=None,
                 initializer=None, activation=None, use_rnn=False, device=None, **kwargs):
        super().__init__()
        self.grouping, self.group_keys = grouping, grouping.group_keys
        self.agent_keys = grouping.agent_keys
        self.n_agents = len(self.agent_keys)
        self.use_rnn = use_rnn
        self.state_space, self.action_space = state_space, action_space
        self.state_dim = int(state_space.shape[0])
        self.n_actions = {k: v.n for k, v in action_space.items()}
        self.joint_action_dim = sum(self.n_actions.values())
        self.representations = representations
        self.representation_info_shape = representations[self.group_keys[0]].output_shapes
        self.critic_head = QValueHead(feature_dim=self.state_dim + self.representation_info_shape['state'][0] +
                                      self.joint_action_dim, hidden_size=critic_hidden_size,
                                      n_actions=max(self.n_actions.values()), normalizer=normalizer,
                                      initializer=initializer, activation=activation, device=device)

    def q_values(self, states, observations, actions, rnn_states=None, return_states=False):
        """states [B, T, S] (or [B, S]), observations [B*n, T, obs] (or [B*n, obs]), actions [B, n, T] (or [B, n]) ->
        Q [R, A] over the (b, i, t) rows."""
        rep = self.representations[self.group_keys[0]](observations, rnn_hidden=rnn_states)
        feat = rep.embeddings
        feat = feat.reshape(-1, feat.shape[-1])
        B = actions.shape[0]
        st = states.reshape(B, -1, self.state_dim)
        acts = actions.reshape(B, self.n_agents, -1)
        q = self.critic_head(critic_input(st, feat, acts, self.n_agents, self.critic_head.n_actions))
        return (q, rep.rnn_states) if return_states else q


class CounterfactualMultiAgentActorCritic(nn.Module):
    """actors + critics + ``target_critics`` (a copy of the critics, refreshed by ``copy_target``)."""

    def __init__(self, grouping, actors, critics, use_rnn=False, device=None, **kwargs):
        super().__init__()
        self.grouping, self.group_keys = grouping, grouping.group_keys
        self.agent_keys = grouping.agent_keys
        self.n_agents = len(self.agent_keys)
        self.actors, self.critics = actors, critics
        self.use_rnn = use_rnn
        self.target_critics = copy.deepcopy(self.critics)

    def logits(self, observations, group=None, rnn_states=None, return_states=False):
        return self.actors[group or self.group_keys[0]].logits(observations, rnn_states, return_states)

    def q_values(self, states, observations, actions, rnn_states=None, return_states=False, target=False):
        critic = self.target_critics if target else self.critics
        return critic.q_values(states, observations, actions, rnn_states, return_states)

    @torch.no_grad()
    def copy_target(self):
        """actor_critic.py:344-346: the critics' parameters into the target critics."""
        for ep, tp in zip(self.critics.parameters(), self.target_critics.parameters()):
            tp.copy_(ep)

    # ---- recurrent states: rows are (env, agent) pairs, as in MultiAgentActorCritic
    def _rnn(self, part):
        g = self.group_keys[0]
        return (self.actors[g].representation if part == "actor" else self.critics.representations[g]).obs_representation

    def init_rnn_states(self, n_rows):
        """Zero actor and critic hidden states [1, n_rows, H] on the device."""
        return self._rnn("actor").init_rnn_states(n_rows), self._rnn("critic").init_rnn_states(n_rows)

    def init_rnn_states_item(self, rows, rnn_states_actor, rnn_states_critic=None):
        """Zero the rows of a finished env in place, on the device."""
        rnn_states_actor[:, rows] = 0.0
        if rnn_states_critic is not None:
            rnn_states_critic[:, rows] = 0.0
        return rnn_states_actor, rnn_states_critic

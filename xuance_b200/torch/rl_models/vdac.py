"""VDAC / IAC model pieces - mirrors of IndependentActorCritic and ValueDecompositionActorCritic
(xuance/torch/rl_models/architectures/multi_agent/actor_critic.py:14-170, 349-379) over the existing CategoricalActor and
StateValueCritic, for one parameter-sharing group.  Module / parameter names follow the reference
(``actors.<group>.representation.obs_representation.*``, ``actors.<group>.actor_head.*``,
``critics.<group>.representation.obs_representation.*``, ``critics.<group>.critic_head.*``, ``v_tot.*`` for the QMIX
mixer), so its ``state_dict`` loads unchanged.

Like the MAPPO model, these work on PACKED rows (one row per agent step, or per agent sequence with ``use_rnn``), and
``logits`` are the raw actor outputs: the action mask is applied by the consumer (K4V, or the acting path)."""
import torch.nn as nn


class IndependentActorCritic(nn.Module):
    def __init__(self, grouping, actors, critics, use_rnn=False, device=None, **kwargs):
        super().__init__()
        self.grouping, self.group_keys = grouping, grouping.group_keys
        self.agent_keys = grouping.agent_keys
        self.n_agents = len(self.agent_keys)
        self.actors, self.critics = actors, critics
        self.use_rnn = use_rnn

    def logits(self, observations, group=None, rnn_states=None, return_states=False):
        return self.actors[group or self.group_keys[0]].logits(observations, rnn_states, return_states)

    def values(self, observations, states=None, group=None, rnn_states=None, return_states=False):
        """Each agent's V_i from its own observation ([rows] or [S, T] with sequences); the critics take no global
        state, so ``states`` is ignored (as by the reference's get_values)."""
        critic = self.critics[group or self.group_keys[0]]
        rep = critic.representation(observations, rnn_hidden=rnn_states)
        out = critic.critic_head(rep.embeddings)
        return (out, rep.rnn_states) if return_states else out

    # ---- recurrent states: rows are (env, agent) pairs, as in MultiAgentActorCritic
    def _rnn(self, part):
        g = self.group_keys[0]
        return (self.actors[g] if part == "actor" else self.critics[g]).representation.obs_representation

    def init_rnn_states(self, n_rows):
        """Zero actor and critic hidden states [1, n_rows, H] on the device."""
        return self._rnn("actor").init_rnn_states(n_rows), self._rnn("critic").init_rnn_states(n_rows)

    def init_rnn_states_item(self, rows, rnn_states_actor, rnn_states_critic=None):
        """Zero the rows of a finished env in place, on the device."""
        rnn_states_actor[:, rows] = 0.0
        if rnn_states_critic is not None:
            rnn_states_critic[:, rows] = 0.0
        return rnn_states_actor, rnn_states_critic


class ValueDecompositionActorCritic(IndependentActorCritic):
    """IndependentActorCritic with a mixer ``v_tot``: VDN_mixer (the sum) or QMIX_Mixer (K9 mix)."""

    def __init__(self, grouping, actors, critics, mixer, use_rnn=False, device=None, **kwargs):
        super().__init__(grouping, actors, critics, use_rnn=use_rnn, device=device)
        self.v_tot = mixer

    def values_tot(self, individual_values, global_states=None):
        """individual_values [rows, n] (agents in key order) -> V_tot [rows, 1]."""
        return self.v_tot(individual_values.reshape(-1, self.n_agents), global_states)

"""DRQN's network: RecurrentQValueHead (xuance/torch/rl_models/heads/q_head.py:126-175) and DeepRecurrentQNetwork
(architectures/single_agent/deep_q_network.py:328-427), with the reference's module and parameter names so its
state_dict loads with strict=True.  The recurrence runs on K13L (``rnn: "LSTM"``, H <= 128) or K13 (``rnn: "GRU"``,
H <= 64); the Q layer is a cuBLAS Linear.  States are RNN_State([1, B, H], [1, B, H] or None) as in the reference."""
from copy import deepcopy

import torch
import torch.nn as nn

from ...common.spaces import is_discrete
from .gru import gru_sequence, check_hidden_size as check_gru_hidden_size
from .layers import mlp_block
from .lstm import lstm_sequence, check_hidden_size as check_lstm_hidden_size
from .outputs import ModelOutput, RNN_State


class RecurrentQValueHead(nn.Module):
    """q_head.py:126-175: ``rnn_layer`` (one-layer batch-first nn.GRU / nn.LSTM, matrices ``initializer``'d, biases
    zero) -> ``q_value`` (one Linear with torch's default initialisation)."""

    def __init__(self, feature_dim, recurrent_hidden_size, recurrent_layer_N, dropout, n_actions, rnn='GRU',
                 initializer=None, device=None, **kwargs):
        super().__init__()
        self.feature_dim, self.n_actions = feature_dim, n_actions
        if rnn == "GRU":
            self.lstm = False
            check_gru_hidden_size(recurrent_hidden_size)
        elif rnn == "LSTM":
            self.lstm = True
            check_lstm_hidden_size(recurrent_hidden_size)
        else:
            raise ValueError("Unknown recurrent module!")
        if recurrent_layer_N != 1:
            raise NotImplementedError("DRQN: recurrent_layer_N = %d is not supported (one recurrent layer)"
                                      % recurrent_layer_N)
        if dropout > 0:
            raise NotImplementedError("DRQN: dropout > 0 is not supported")
        cls = nn.LSTM if self.lstm else nn.GRU
        self.rnn_layer = cls(input_size=feature_dim, hidden_size=recurrent_hidden_size, num_layers=1, batch_first=True,
                             device=device)
        if initializer is not None:
            for weight_list in self.rnn_layer.all_weights:
                for w in weight_list:
                    initializer(w) if len(w.shape) > 1 else nn.init.constant_(w, 0)
        self.q_value = nn.Sequential(*mlp_block(recurrent_hidden_size, n_actions, None, None, None, device)[0])

    def forward(self, features, rnn_states=None, avail_actions=None, **kwargs):
        """features [B, T, F]; rnn_states None (zeros) or RNN_State of [1, B, H] -> (RNN_State, q [B, T, A])."""
        B, H = features.shape[0], self.rnn_layer.hidden_size
        h0 = c0 = None
        if rnn_states is not None:
            h0 = rnn_states.hidden_states.reshape(B, H)
            c0 = rnn_states.cell_states.reshape(B, H) if self.lstm else None
        if self.lstm:
            y, hT, cT = lstm_sequence(self.rnn_layer, features, h0, c0)
            out = RNN_State(hidden_states=hT.unsqueeze(0), cell_states=cT.unsqueeze(0))
        else:
            y, hT = gru_sequence(self.rnn_layer, features, h0)
            out = RNN_State(hidden_states=hT.unsqueeze(0))
        q = self.q_value(y)
        if avail_actions is not None:
            q = q.masked_fill(avail_actions == 0, -1e10)
        return out, q


class DeepRecurrentQNetwork(nn.Module):
    """deep_q_network.py:328-427: eval representation + recurrent Q head and their deep-copied targets."""

    def __init__(self, representation, recurrent_hidden_size, recurrent_layer_N, dropout, action_space=None, rnn='GRU',
                 initializer=None, device=None, use_distributed_training=False, **kwargs):
        super().__init__()
        if not is_discrete(action_space):
            raise ValueError('action_space must be Discrete')
        if use_distributed_training:
            raise NotImplementedError("DRQN: distributed training is not supported (one rank)")
        self.n_actions = action_space.n
        self.device = device
        self.representation = representation
        self.target_representation = deepcopy(representation)
        self.representation_info_shape = representation.output_shapes
        self.recurrent_layer_N = recurrent_layer_N
        self.recurrent_hidden_size = recurrent_hidden_size
        self.eval_Q_head = RecurrentQValueHead(feature_dim=self.representation_info_shape['state'][0],
                                               recurrent_hidden_size=recurrent_hidden_size,
                                               recurrent_layer_N=recurrent_layer_N, dropout=dropout,
                                               n_actions=self.n_actions, rnn=rnn, initializer=initializer, device=device)
        self.target_Q_head = deepcopy(self.eval_Q_head)
        self.lstm = self.eval_Q_head.lstm
        self.distributed_training = False

    def eval_parameters(self):
        return list(self.representation.parameters()) + list(self.eval_Q_head.parameters())

    def target_parameters(self):
        return list(self.target_representation.parameters()) + list(self.target_Q_head.parameters())

    def forward(self, observation, rnn_states=None, **kwargs):
        """observation [B, T, obs] -> (RNN_State, ModelOutput(actions = greedy action at the last step, values = Q))."""
        rep = self.representation(observation)
        rnn_new, q = self.eval_Q_head(rep.embeddings, rnn_states)
        return rnn_new, ModelOutput(actions=q[:, -1].argmax(dim=-1), values=q, rep_out=rep)

    def target(self, observation, rnn_states=None, **kwargs):
        rep = self.target_representation(observation)
        rnn_new, q = self.target_Q_head(rep.embeddings, rnn_states)
        return rnn_new, ModelOutput(actions=q.argmax(dim=-1), values=q)

    def init_rnn_states(self, batch):
        h = torch.zeros((self.recurrent_layer_N, batch, self.recurrent_hidden_size), device=self.device)
        return RNN_State(hidden_states=h, cell_states=torch.zeros_like(h) if self.lstm else None)

    def init_rnn_states_item(self, rnn_states, i):
        rnn_states.hidden_states[:, i] = 0.0
        if self.lstm:
            rnn_states.cell_states[:, i] = 0.0
        return rnn_states

    def copy_target(self):
        for ep, tp in zip(self.representation.parameters(), self.target_representation.parameters()):
            tp.data.copy_(ep)
        for ep, tp in zip(self.eval_Q_head.parameters(), self.target_Q_head.parameters()):
            tp.data.copy_(ep)

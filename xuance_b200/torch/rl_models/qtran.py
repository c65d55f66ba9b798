"""QTRAN model pieces (reference: heads/q_mix_head.py:143-289, architectures/multi_agent/value_factorization.py:321-446).
Module and parameter names mirror the reference so its ``state_dict`` loads with strict=True.  Scope: one
parameter-sharing group of K13 GRU agents (use_rnn=True).

Q_jt and V_jt are torch Linear layers (cuBLAS GEMMs).  The input assembly of Q_jt - the masked hidden states, the one-hot
actions, the shared ``action_encoding`` MLP, the sum over agents (base) or, as the reference's QTRAN_Alt computes it, n-1 copies of each agent's own
encoding and the agent ids (alt),
the state columns - is K9Q (``xb_qtran_encode_fwd``), forward and backward."""
from copy import deepcopy

import torch
import torch.nn as nn

from ... import _lib
from .qmix import MixingQNetwork, VDN_mixer

MAX_AGENTS, MAX_ACTIONS, MAX_HIDDEN = 32, 64, 64   # K9Q's limits (include/xb200.h)
BASE, ALT = 0, 1


def check_limits(n, A, H):
    if n > MAX_AGENTS or A > MAX_ACTIONS or H > MAX_HIDDEN:
        raise NotImplementedError("QTRAN kernels: %d agents, %d actions and hidden size %d are outside the supported "
                                  "n <= %d, A <= %d, H <= %d" % (n, A, H, MAX_AGENTS, MAX_ACTIONS, MAX_HIDDEN))


class QTRAN_Base(nn.Module):
    """q_mix_head.py:143-211: Q_jt on [state, sum_i action_encoding([h_i, onehot(a_i)])], V_jt on the state."""
    mode = BASE

    def __init__(self, dim_state=0, action_space=None, dim_hidden=32, n_agents=1, dim_utility_hidden=1,
                 use_parameter_sharing=False, device=None):
        super().__init__()
        self.dim_state, self.action_space, self.dim_hidden, self.n_agents = dim_state, action_space, dim_hidden, n_agents
        self.n_actions_max = max(a.n for a in action_space.values())
        self.use_parameter_sharing, self.device = use_parameter_sharing, device
        self.dim_ae_input = dim_utility_hidden + self.n_actions_max
        self.dim_q_input = dim_state + self.dim_ae_input + (n_agents if self.mode == ALT else 0)
        self.dim_v_input = dim_state
        q_out = self.n_actions_max if self.mode == ALT else 1
        self.Q_jt = nn.Sequential(nn.Linear(self.dim_q_input, dim_hidden), nn.ReLU(), nn.Linear(dim_hidden, dim_hidden),
                                  nn.ReLU(), nn.Linear(dim_hidden, q_out)).to(device)
        self.V_jt = nn.Sequential(nn.Linear(self.dim_v_input, dim_hidden), nn.ReLU(), nn.Linear(dim_hidden, dim_hidden),
                                  nn.ReLU(), nn.Linear(dim_hidden, 1)).to(device)
        self.action_encoding = nn.Sequential(nn.Linear(self.dim_ae_input, self.dim_ae_input), nn.ReLU(),
                                             nn.Linear(self.dim_ae_input, self.dim_ae_input)).to(device)

    def encode(self, states, state_t0, h, agent_mask, actions):
        """The Q_jt input: see ``qtran_encode``."""
        enc = self.action_encoding
        return qtran_encode(self.mode, states, state_t0, h, agent_mask, actions, enc[0].weight, enc[0].bias,
                            enc[2].weight, enc[2].bias)


class QTRAN_Alt(QTRAN_Base):
    """q_mix_head.py:214-289: one Q_jt row per agent i, [state, (n-1) * encoding_i, onehot_n(i)] -> A values.  The
    reference masks the repeat axis of agent i's own encoding, so the "sum across other agents" is n-1 copies of e_i."""
    mode = ALT


class _EncodeFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, w1, b1, w2, b2, states, state_t0, agent_mask, actions, mode, train):
        B, n, T1, H = h.shape
        T, S, D = agent_mask.shape[2], states.shape[-1], w1.shape[0]
        A = D - H
        rows, width = (B * T * n, S + D + n) if mode == ALT else (B * T, S + D)
        x = torch.empty((rows, width), dtype=torch.float32, device=h.device)
        pre = torch.empty((B * T * n, D), dtype=torch.float32, device=h.device) if train else None
        act_f, act_i = (actions, None) if actions.dtype == torch.float32 else (None, actions)
        _lib.call("xb_qtran_encode_fwd", mode, _lib.ptr(states), state_t0, _lib.ptr(h), _lib.ptr(agent_mask),
                  _lib.ptr(act_f), _lib.ptr(act_i), actions.shape[2], _lib.ptr(w1), _lib.ptr(b1), _lib.ptr(w2),
                  _lib.ptr(b2), B, n, T, S, H, A, _lib.ptr(x), _lib.ptr(pre))
        if train:
            ctx.save_for_backward(h, w1, w2, pre, agent_mask, actions)
            ctx.dims = (mode, B, n, T, S, H, A)
        return x

    @staticmethod
    def backward(ctx, dx):
        h, w1, w2, pre, agent_mask, actions = ctx.saved_tensors
        mode, B, n, T, S, H, A = ctx.dims
        dev = h.device
        dh = torch.empty_like(h)
        dw1, dw2 = torch.empty_like(w1), torch.empty_like(w2)
        db1 = torch.empty(w1.shape[0], dtype=torch.float32, device=dev)
        db2 = torch.empty_like(db1)
        need = int(_lib.load().xb_qtran_encode_bwd_work(B, n, T, H, A))
        work = torch.empty(need, dtype=torch.float32, device=dev)
        act_f, act_i = (actions, None) if actions.dtype == torch.float32 else (None, actions)
        _lib.call("xb_qtran_encode_bwd", mode, _lib.ptr(dx.contiguous()), _lib.ptr(h), _lib.ptr(agent_mask),
                  _lib.ptr(act_f), _lib.ptr(act_i), actions.shape[2], _lib.ptr(w1), _lib.ptr(w2), _lib.ptr(pre), B, n,
                  T, S, H, A, _lib.ptr(dh), _lib.ptr(dw1), _lib.ptr(db1), _lib.ptr(dw2), _lib.ptr(db2), _lib.ptr(work),
                  need)
        return dh, dw1, db1, dw2, db2, None, None, None, None, None, None


def qtran_encode(mode, states, state_t0, h, agent_mask, actions, w1, b1, w2, b2):
    """K9Q encoder: states [B, T+1, S] read at steps state_t0 + t; h [B, n, T+1, H] (GRU outputs) at steps 0..T-1;
    agent_mask [B, n, T]; actions [B, n, >= T] float32 or int32 -> the Q_jt input [B*T, S+D] (base) or
    [B*T*n, S+D+n] (alt), D = H + A.  Differentiable in h and the encoder's weights."""
    train = torch.is_grad_enabled() and any(t.requires_grad for t in (h, w1, b1, w2, b2))
    return _EncodeFunction.apply(h, w1.contiguous(), b1, w2.contiguous(), b2, states.contiguous(), state_t0,
                                 agent_mask, actions.contiguous(), mode, train)


class QTranMixingNetwork(MixingQNetwork):
    """value_factorization.py:321-446 for one shared group: the agent networks (K13 GRU agents) and their target copy,
    the VDN eval_Qtot / target_Qtot, qtran_net and target_qtran_net, registered in the reference's order."""

    def __init__(self, grouping, q_networks, mixer, qtran_mixer, use_rnn=True, device=None, **kwargs):
        super().__init__(grouping, q_networks, mixer if mixer is not None else VDN_mixer(), use_rnn=use_rnn,
                         device=device, **kwargs)
        self.n_actions = {k: self.individual_q_networks[k].action_space.n for k in self.group_keys}
        self.n_actions_max = max(self.n_actions.values())
        self.qtran_net = qtran_mixer
        self.target_qtran_net = deepcopy(qtran_mixer)

    @property
    def parameters_model(self):
        return list(self.qtran_net.parameters()) + list(self.eval_Qtot.parameters()) + \
            list(self.individual_q_networks.parameters())

    def q_and_hidden(self, packed_obs, target=False):
        """packed_obs [B*n, T+1, obs] -> (Q [B*n, T+1, A], GRU outputs [B*n, T+1, H]) from a zero initial state."""
        net = (self.target_individual_q_networks if target else self.individual_q_networks)[self.group_keys[0]]
        q, rep = net(packed_obs)
        return q, rep.embeddings

    def copy_target(self):
        super().copy_target()
        for ep, tp in zip(self.qtran_net.parameters(), self.target_qtran_net.parameters()):
            tp.data.copy_(ep)

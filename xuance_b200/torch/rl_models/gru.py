"""The recurrence of a one-layer GRU on K13 (``xb_gru_seq_fwd`` / ``xb_gru_seq_bwd``), and the LayerNorm variant of
``Basic_RNN`` (xuance/torch/rl_models/representations/rnn.py:9-99) that runs on it.

``gru_sequence`` keeps torch.nn.GRU's arithmetic split: the input projection ``x W_ih^T + b_ih`` for all T at once is a
cuBLAS GEMM through torch (so dx, dW_ih and db_ih are torch's Linear backward), K13 walks the time steps, and the
backward's ``dW_hh = sum dgh^T h_{t-1}`` / ``db_hh = sum dgh`` are one GEMM and one sum.  Acting runs the same forward
kernel with T = 1 and a carried state, so a rollout step and step t of the training forward execute the same code.

QMIX keeps its cuDNN ``Basic_RNN`` (rl_models/qmix.py); moving it onto K13 would change its numerics."""
from types import SimpleNamespace

import torch
import torch.nn as nn

from ... import _lib
from .layers import mlp_block
from .outputs import RepresentationOutput

MAX_HIDDEN = 64   # K13 keeps W_hh [3H, H] resident in shared memory: 48 KB at H = 64


def check_hidden_size(H, name="K13 GRU sequence kernels"):
    if not 1 <= H <= MAX_HIDDEN:
        raise NotImplementedError("%s: recurrent_hidden_size %d is outside the supported 1..%d"
                                  % (name, H, MAX_HIDDEN))


def check_scope(name, config):
    """Refuse a recurrent representation K13 does not run, naming ``name`` (the algorithm) in the error: K13 runs one
    GRU layer of 1..MAX_HIDDEN units without dropout.  ``config`` has ``recurrent_hidden_size`` and may have ``rnn``,
    ``N_recurrent_layers`` and ``dropout`` (defaults GRU, 1, 0)."""
    if getattr(config, "rnn", "GRU") != "GRU":
        raise NotImplementedError("%s: LSTM representations are not supported (GRU only)" % name)
    if getattr(config, "N_recurrent_layers", 1) != 1:
        raise NotImplementedError("%s: N_recurrent_layers > 1 is not supported (one GRU layer)" % name)
    if getattr(config, "dropout", 0) > 0:
        raise NotImplementedError("%s: dropout > 0 is not supported" % name)
    check_hidden_size(config.recurrent_hidden_size, name)


class GRUSequence(torch.autograd.Function):
    """(xg [S, T, 3H], w_hh [3H, H], b_hh [3H], h0 [S, H] or None) -> (y [S, T, H], hT [S, H])."""

    @staticmethod
    def forward(ctx, xg, w_hh, b_hh, h0):
        S, T, G = xg.shape
        H = G // 3
        check_hidden_size(H)
        xg, w_hh, b_hh = xg.contiguous(), w_hh.contiguous(), b_hh.contiguous()
        h0 = None if h0 is None else h0.contiguous()
        y = torch.empty((S, T, H), dtype=torch.float32, device=xg.device)
        hT = torch.empty((S, H), dtype=torch.float32, device=xg.device)
        train = any(ctx.needs_input_grad)     # grad mode is off inside forward; an inference call saves nothing
        gates = torch.empty((S, T, 4 * H), dtype=torch.float32, device=xg.device) if train else None
        _lib.call("xb_gru_seq_fwd", _lib.ptr(xg), _lib.ptr(w_hh), _lib.ptr(b_hh), _lib.ptr(h0), S, T, H, _lib.ptr(y),
                  _lib.ptr(hT), _lib.ptr(gates))
        if gates is not None:
            ctx.save_for_backward(w_hh, gates, y, h0)
        return y, hT

    @staticmethod
    def backward(ctx, dy, dhT):
        w_hh, gates, y, h0 = ctx.saved_tensors
        S, T, H = y.shape
        dy = dy.contiguous()
        dhT = None if dhT is None else dhT.contiguous()
        dxg = torch.empty((S, T, 3 * H), dtype=torch.float32, device=y.device)
        dgh = torch.empty_like(dxg)
        dh0 = torch.empty((S, H), dtype=torch.float32, device=y.device) if ctx.needs_input_grad[3] else None
        _lib.call("xb_gru_seq_bwd", _lib.ptr(dy), _lib.ptr(dhT), _lib.ptr(w_hh), _lib.ptr(gates), _lib.ptr(y),
                  _lib.ptr(h0), S, T, H, _lib.ptr(dxg), _lib.ptr(dgh), _lib.ptr(dh0))
        dw_hh = db_hh = None
        if ctx.needs_input_grad[1]:
            h_prev = torch.cat([h0.unsqueeze(1) if h0 is not None else y.new_zeros(S, 1, H), y[:, :-1]], dim=1)
            dw_hh = dgh.reshape(-1, 3 * H).t().mm(h_prev.reshape(-1, H))
        if ctx.needs_input_grad[2]:
            db_hh = dgh.reshape(-1, 3 * H).sum(dim=0)
        return dxg, dw_hh, db_hh, dh0


def gru_sequence(gru, x, h0=None):
    """One-layer batch-first ``gru`` (an nn.GRU, used as the parameter container) over x [S, T, I] from h0 [S, H] (None:
    zeros) -> (y [S, T, H], hT [S, H])."""
    xg = torch.nn.functional.linear(x, gru.weight_ih_l0, gru.bias_ih_l0)
    return GRUSequence.apply(xg, gru.weight_hh_l0, gru.bias_hh_l0, h0)


class Basic_RNN_K13(nn.Module):
    """rnn.py:9-99, GRU variant, for MAPPO: ``input_norm`` (LayerNorm on the observation) -> ``mlp`` (Linear, activation,
    LayerNorm per layer) -> one-layer GRU (``rnn``, orthogonal weights and zero biases, recurrence on K13) ->
    ``norm_rnn`` (LayerNorm on the GRU output).  Module and parameter names are the reference's, so its state_dict loads
    with strict=True.  Inputs are [S, T, obs] (or [S, obs] for one step); states are [1, S, H] like the reference's."""

    def __init__(self, input_shape, hidden_sizes=None, normalize=None, initialize=None, activation=None, device=None,
                 **kwargs):
        super().__init__()
        check_scope("Basic_RNN_K13", SimpleNamespace(**kwargs))
        self.input_shape = input_shape
        self.fc_hidden_sizes = kwargs["fc_hidden_sizes"]
        self.recurrent_hidden_size = kwargs["recurrent_hidden_size"]
        self.N_recurrent_layer = 1
        self.lstm = False
        self.normalize, self.device = normalize, device
        self.output_shapes = {'state': (self.recurrent_hidden_size,)}
        layers, shape = [], input_shape
        for h in self.fc_hidden_sizes:
            blk, shape = mlp_block(shape[0], h, normalize, activation, initialize, device=device)
            layers.extend(blk)
        self.mlp = nn.Sequential(*layers)
        self.rnn = nn.GRU(input_size=shape[0], hidden_size=self.recurrent_hidden_size, num_layers=1, batch_first=True,
                          device=device)
        if initialize is not None:
            for wl in self.rnn.all_weights:
                for w in wl:
                    initialize(w) if len(w.shape) > 1 else nn.init.constant_(w, 0)
        self.use_normalize = normalize is not None
        if self.use_normalize:
            self.input_norm = normalize(input_shape, device=device)
            self.norm_rnn = normalize(self.recurrent_hidden_size, device=device)

    def forward(self, x, rnn_hidden=None, **kwargs):
        """x [S, T, obs] or [S, obs]; rnn_hidden [1, S, H] or None (zeros).  embeddings [S, T, H] ([S, H] for 2-D x)."""
        x = torch.as_tensor(x, dtype=torch.float32, device=self.device)
        one_step = x.dim() == 2
        if one_step:
            x = x.unsqueeze(1)
        if self.use_normalize:
            x = self.input_norm(x)
        h0 = None if rnn_hidden is None else rnn_hidden.reshape(x.shape[0], self.recurrent_hidden_size)
        y, hT = gru_sequence(self.rnn, self.mlp(x), h0)
        if self.use_normalize:
            y = self.norm_rnn(y)
        return RepresentationOutput(embeddings=y[:, 0] if one_step else y, rnn_states=hT.detach().unsqueeze(0))

    def init_rnn_states(self, batch):
        return torch.zeros((1, batch, self.recurrent_hidden_size), device=self.device)

    def init_rnn_states_item(self, indexes, rnn_states):
        rnn_states[:, indexes] = 0.0
        return rnn_states

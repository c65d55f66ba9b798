"""The recurrence of a one-layer LSTM on K13L (``xb_lstm_seq_fwd`` / ``xb_lstm_seq_bwd``).

``lstm_sequence`` keeps torch.nn.LSTM's arithmetic split as ``gru_sequence`` does: the input projection
``x W_ih^T + b_ih`` for all T at once is a cuBLAS GEMM through torch (so dx, dW_ih and db_ih are torch's Linear
backward), K13L walks the time steps, and the backward's ``dW_hh = sum dgates^T h_{t-1}`` / ``db_hh = sum dgates`` are
one GEMM and one sum.  Acting runs the same forward kernel with T = 1 and a carried (h, c), so an acting step and step t
of the training forward execute the same code."""
import torch

from ... import _lib

MAX_HIDDEN = 128   # K13L keeps W_hh [4H, H] on chip: registers plus 192 KB of shared memory at H = 128


def check_hidden_size(H):
    if not 1 <= H <= MAX_HIDDEN:
        raise NotImplementedError("K13L LSTM sequence kernels: recurrent_hidden_size %d is outside the supported 1..%d"
                                  % (H, MAX_HIDDEN))


class LSTMSequence(torch.autograd.Function):
    """(xg [S, T, 4H], w_hh [4H, H], b_hh [4H], h0, c0 [S, H] or None) -> (y [S, T, H], hT [S, H], cT [S, H])."""

    @staticmethod
    def forward(ctx, xg, w_hh, b_hh, h0, c0):
        S, T, G = xg.shape
        H = G // 4
        check_hidden_size(H)
        xg, w_hh, b_hh = xg.contiguous(), w_hh.contiguous(), b_hh.contiguous()
        h0 = None if h0 is None else h0.contiguous()
        c0 = None if c0 is None else c0.contiguous()
        y = torch.empty((S, T, H), dtype=torch.float32, device=xg.device)
        hT = torch.empty((S, H), dtype=torch.float32, device=xg.device)
        cT = torch.empty((S, H), dtype=torch.float32, device=xg.device)
        train = any(ctx.needs_input_grad)     # grad mode is off inside forward; an inference call saves nothing
        gates = torch.empty((S, T, 5 * H), dtype=torch.float32, device=xg.device) if train else None
        _lib.call("xb_lstm_seq_fwd", _lib.ptr(xg), _lib.ptr(w_hh), _lib.ptr(b_hh), _lib.ptr(h0), _lib.ptr(c0), S, T, H,
                  _lib.ptr(y), _lib.ptr(hT), _lib.ptr(cT), _lib.ptr(gates))
        if gates is not None:
            ctx.save_for_backward(w_hh, gates, y, h0, c0)
        return y, hT, cT

    @staticmethod
    def backward(ctx, dy, dhT, dcT):
        w_hh, gates, y, h0, c0 = ctx.saved_tensors
        S, T, H = y.shape
        dy = dy.contiguous()
        dhT = None if dhT is None else dhT.contiguous()
        dcT = None if dcT is None else dcT.contiguous()
        dxg = torch.empty((S, T, 4 * H), dtype=torch.float32, device=y.device)
        dh0 = torch.empty((S, H), dtype=torch.float32, device=y.device) if ctx.needs_input_grad[3] else None
        dc0 = torch.empty((S, H), dtype=torch.float32, device=y.device) if ctx.needs_input_grad[4] else None
        _lib.call("xb_lstm_seq_bwd", _lib.ptr(dy), _lib.ptr(dhT), _lib.ptr(dcT), _lib.ptr(w_hh), _lib.ptr(gates),
                  _lib.ptr(c0), S, T, H, _lib.ptr(dxg), _lib.ptr(dh0), _lib.ptr(dc0))
        dw_hh = db_hh = None
        if ctx.needs_input_grad[1]:
            h_prev = torch.cat([h0.unsqueeze(1) if h0 is not None else y.new_zeros(S, 1, H), y[:, :-1]], dim=1)
            dw_hh = dxg.reshape(-1, 4 * H).t().mm(h_prev.reshape(-1, H))
        if ctx.needs_input_grad[2]:
            db_hh = dxg.reshape(-1, 4 * H).sum(dim=0)
        return dxg, dw_hh, db_hh, dh0, dc0


def lstm_sequence(lstm, x, h0=None, c0=None):
    """One-layer batch-first ``lstm`` (an nn.LSTM, used as the parameter container) over x [S, T, I] from h0, c0 [S, H]
    (None: zeros) -> (y [S, T, H], hT [S, H], cT [S, H])."""
    xg = torch.nn.functional.linear(x, lstm.weight_ih_l0, lstm.bias_ih_l0)
    return LSTMSequence.apply(xg, lstm.weight_hh_l0, lstm.bias_hh_l0, h0, c0)

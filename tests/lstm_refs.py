"""float64 restatement of K13L (xb_lstm_seq_fwd / xb_lstm_seq_bwd): the recurrence of a one-layer torch.nn.LSTM (gate
order i, f, g, o) split the way the kernels split it.  The forward takes the projected input xg = x W_ih^T + b_ih and
returns y, hT, cT and the saved gates {i, f, g, o, c}; the backward returns dxg (the gradient of the pre-activations,
which is also the gradient of W_hh h + b_hh), dh0 and dc0.  test_drqn.py pins these against torch.nn.LSTM autograd in
float64."""
import numpy as np


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def lstm_fwd(xg, w_hh, b_hh, h0=None, c0=None):
    """xg [S, T, 4H], w_hh [4H, H], b_hh [4H], h0 / c0 [S, H] or None -> y [S, T, H], hT, cT [S, H], gates [S, T, 5H]."""
    xg, w_hh, b_hh = (np.asarray(a, np.float64) for a in (xg, w_hh, b_hh))
    S, T, G = xg.shape
    H = G // 4
    h = np.zeros((S, H)) if h0 is None else np.asarray(h0, np.float64).copy()
    c = np.zeros((S, H)) if c0 is None else np.asarray(c0, np.float64).copy()
    y = np.empty((S, T, H))
    gates = np.empty((S, T, 5 * H))
    for t in range(T):
        pre = xg[:, t] + (h @ w_hh.T + b_hh)
        i, f = _sigmoid(pre[:, :H]), _sigmoid(pre[:, H:2 * H])
        g, o = np.tanh(pre[:, 2 * H:3 * H]), _sigmoid(pre[:, 3 * H:])
        c = f * c + i * g
        h = o * np.tanh(c)
        y[:, t] = h
        gates[:, t] = np.concatenate([i, f, g, o, c], axis=1)
    return y, h.copy(), c.copy(), gates


def lstm_bwd(dy, dhT, dcT, w_hh, gates, c0=None):
    """dy [S, T, H], dhT / dcT [S, H] or None, the forward's gates -> dxg [S, T, 4H], dh0, dc0 [S, H]."""
    dy, w_hh, gates = (np.asarray(a, np.float64) for a in (dy, w_hh, gates))
    S, T, H = dy.shape
    dh_next = np.zeros((S, H)) if dhT is None else np.asarray(dhT, np.float64).copy()
    dc = np.zeros((S, H)) if dcT is None else np.asarray(dcT, np.float64).copy()
    dxg = np.empty((S, T, 4 * H))
    for t in range(T - 1, -1, -1):
        i, f, g, o, c = (gates[:, t, k * H:(k + 1) * H] for k in range(5))
        cp = gates[:, t - 1, 4 * H:] if t > 0 else (np.zeros((S, H)) if c0 is None else np.asarray(c0, np.float64))
        dh = dh_next + dy[:, t]
        tc = np.tanh(c)
        dc = dc + dh * o * (1.0 - tc * tc)
        d = np.concatenate([dc * g * i * (1 - i), dc * cp * f * (1 - f), dc * i * (1 - g * g), dh * tc * o * (1 - o)], 1)
        dxg[:, t] = d
        dc = dc * f
        dh_next = d @ w_hh
    return dxg, dh_next, dc


def lstm_param_grads(x, dxg, y, h0=None):
    """The GEMM half of the backward: dW_ih, db_ih, dW_hh, db_hh from dxg, the inputs x and the outputs y."""
    x, dxg, y = (np.asarray(a, np.float64) for a in (x, dxg, y))
    S, T, H = y.shape
    hp = np.concatenate([np.zeros((S, 1, H)) if h0 is None else np.asarray(h0, np.float64)[:, None], y[:, :-1]], 1)
    d2 = dxg.reshape(-1, 4 * H)
    return {"dW_ih": d2.T @ x.reshape(S * T, -1), "db_ih": d2.sum(0), "dW_hh": d2.T @ hp.reshape(S * T, H),
            "db_hh": d2.sum(0)}

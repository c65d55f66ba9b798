"""float64 restatement of K13 (xb_gru_seq_fwd / xb_gru_seq_bwd): the recurrence of a one-layer torch.nn.GRU split the way
the kernels split it.  The forward takes the projected input xg = x W_ih^T + b_ih and returns y, hT and the saved gates
{r, z, n, gh_n}; the backward returns dxg (the gradient of xg), dgh (the gradient of W_hh h + b_hh) and dh0.
test_mappo_rnn.py pins these against torch.nn.GRU autograd in float64."""
import numpy as np


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def gru_fwd(xg, w_hh, b_hh, h0=None):
    """xg [S, T, 3H], w_hh [3H, H], b_hh [3H], h0 [S, H] or None -> y [S, T, H], hT [S, H], gates [S, T, 4H]."""
    xg, w_hh, b_hh = (np.asarray(a, np.float64) for a in (xg, w_hh, b_hh))
    S, T, G = xg.shape
    H = G // 3
    h = np.zeros((S, H)) if h0 is None else np.asarray(h0, np.float64).copy()
    y = np.empty((S, T, H))
    gates = np.empty((S, T, 4 * H))
    for t in range(T):
        gh = h @ w_hh.T + b_hh
        r = _sigmoid(xg[:, t, :H] + gh[:, :H])
        z = _sigmoid(xg[:, t, H:2 * H] + gh[:, H:2 * H])
        n = np.tanh(xg[:, t, 2 * H:] + r * gh[:, 2 * H:])
        h = (1.0 - z) * n + z * h
        y[:, t] = h
        gates[:, t] = np.concatenate([r, z, n, gh[:, 2 * H:]], axis=1)
    return y, h.copy(), gates


def gru_bwd(dy, dhT, w_hh, gates, y, h0=None):
    """-> dxg [S, T, 3H], dgh [S, T, 3H], dh0 [S, H]."""
    dy, w_hh, gates, y = (np.asarray(a, np.float64) for a in (dy, w_hh, gates, y))
    S, T, H = y.shape
    dh = np.zeros((S, H)) if dhT is None else np.asarray(dhT, np.float64).copy()
    dxg = np.empty((S, T, 3 * H))
    dgh = np.empty((S, T, 3 * H))
    for t in range(T - 1, -1, -1):
        dh = dh + dy[:, t]
        r, z, n, hn = (gates[:, t, k * H:(k + 1) * H] for k in range(4))
        hp = y[:, t - 1] if t > 0 else (np.zeros((S, H)) if h0 is None else np.asarray(h0, np.float64))
        dnp = dh * (1.0 - z) * (1.0 - n * n)
        dzp = dh * (hp - n) * z * (1.0 - z)
        drp = dnp * hn * r * (1.0 - r)
        dxg[:, t] = np.concatenate([drp, dzp, dnp], axis=1)
        dgh[:, t] = np.concatenate([drp, dzp, dnp * r], axis=1)
        dh = dh * z + dgh[:, t] @ w_hh
    return dxg, dgh, dh


def gru_param_grads(x, dxg, dgh, y, h0=None):
    """The time-independent gradients the caller forms with GEMMs: dx, dW_ih, db_ih (from dxg), dW_hh, db_hh (from dgh)."""
    x = np.asarray(x, np.float64)
    S, T, H = y.shape
    hp = np.concatenate([(np.zeros((S, 1, H)) if h0 is None else np.asarray(h0, np.float64)[:, None]), y[:, :-1]], 1)
    G = 3 * H
    return {"dW_ih": dxg.reshape(-1, G).T @ x.reshape(S * T, -1), "db_ih": dxg.reshape(-1, G).sum(0),
            "dW_hh": dgh.reshape(-1, G).T @ hp.reshape(-1, H), "db_hh": dgh.reshape(-1, G).sum(0)}

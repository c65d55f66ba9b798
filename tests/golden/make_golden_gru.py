"""Generate tests/golden/gru_basic_rnn.npz by running the UNMODIFIED reference (agi-brain/xuance v1.4.4 @ 4f0b05b).

Run in the build container only (needs /root/reference):   python tests/golden/make_golden_gru.py

The reference's Basic_RNN (representations/rnn.py:9-99) as recurrent MAPPO's SMAC configs build it: LayerNorm
normalisation, orthogonal initialisation, ReLU, fc_hidden_sizes [64], one GRU layer of 64, input 30 (SMAC 3m).  Records
its freshly initialised state_dict (keys, shapes and the reference's initialisation), one forward over [6, 9, 30] from a
nonzero initial state (float32 on the CPU) and the parameter / input gradients of sum(embeddings * w)."""
import os

import numpy as np
import torch
import torch.nn as nn

from make_golden import ENV, HERE  # noqa: E402  (imports the reference and sets up sys.path)
from xuance.torch.rl_models.representations.rnn import Basic_RNN  # noqa: E402
from xuance.torch.rl_models.modules.outputs import RNN_State  # noqa: E402

OBS, FC, H, S, T = 30, 64, 64, 6, 9


def main():
    torch.manual_seed(0)
    rep = Basic_RNN((OBS,), None, normalize=nn.LayerNorm, initialize=nn.init.orthogonal_, activation=nn.ReLU,
                    device="cpu", fc_hidden_sizes=[FC], recurrent_hidden_size=H, N_recurrent_layers=1, dropout=0,
                    rnn="GRU")
    # LayerNorm affine parameters start at 1 / 0; move them so the fixture pins that they are applied
    with torch.no_grad():
        for m in rep.modules():
            if isinstance(m, nn.LayerNorm):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
    out = {"env": ENV, "dims": np.array([OBS, FC, H, S, T])}
    for k, v in rep.state_dict().items():
        out["sd/" + k] = v.numpy().copy()
    rng = np.random.default_rng(13)
    x = torch.tensor(rng.standard_normal((S, T, OBS)).astype(np.float32), requires_grad=True)
    h0 = torch.tensor((0.5 * rng.standard_normal((1, S, H))).astype(np.float32), requires_grad=True)
    w = torch.tensor(rng.standard_normal((S, T, H)).astype(np.float32))
    o = rep(x, RNN_State(hidden_states=h0))
    (o.embeddings * w).sum().backward()
    out.update({"x": x.detach().numpy(), "h0": h0.detach().numpy(), "w": w.numpy(),
                "embeddings": o.embeddings.detach().numpy(), "hn": o.rnn_states.hidden_states.numpy(),
                "grad/x": x.grad.numpy(), "grad/h0": h0.grad.numpy()})
    for k, p in rep.named_parameters():
        out["grad/" + k] = p.grad.numpy().copy()
    np.savez_compressed(os.path.join(HERE, "gru_basic_rnn.npz"), **out)


if __name__ == "__main__":
    main()

"""torch-CPU oracle of the recurrent MAPPO model: a copy of the device model's parameters in which each Basic_RNN_K13
runs its GRU through nn.GRU on the CPU (no K13, no cuDNN).  With tests/oracle_mappo.py's MAPPOLearnerOracle (torch
autograd of the reference's loss, torch Adam) it restates the recurrent MAPPO_Learner.update over [B*n, T] sequences."""
import copy

import torch.nn as nn


class CPUBasicRNN(nn.Module):
    """Oracle stand-in for Basic_RNN_K13: the same modules, with the GRU run by nn.GRU on the CPU."""

    def __init__(self, k13):
        super().__init__()
        self.input_norm, self.mlp = copy.deepcopy(k13.input_norm), copy.deepcopy(k13.mlp)
        self.rnn, self.norm_rnn = copy.deepcopy(k13.rnn), copy.deepcopy(k13.norm_rnn)
        self.output_shapes = k13.output_shapes

    def forward(self, x, rnn_hidden=None, **kwargs):
        from xuance_b200.torch.rl_models.outputs import RepresentationOutput
        y, hn = self.rnn(self.mlp(self.input_norm(x)), rnn_hidden)
        return RepresentationOutput(embeddings=self.norm_rnn(y), rnn_states=hn)


class RecurrentModelOracle(nn.Module):
    """The device model's parameters on the CPU, GRUs on nn.GRU; outputs flattened to rows as the learner's are."""

    def __init__(self, model):
        super().__init__()
        self.m = copy.deepcopy(model).cpu()
        for part in (self.m.actors["shared"].representation, self.m.critics["shared"].representations["shared"]):
            part.obs_representation = CPUBasicRNN(part.obs_representation)

    def logits(self, obs):
        out = self.m.logits(obs)
        return out.reshape(-1, out.shape[-1])

    def values(self, obs, states=None):
        return self.m.values(obs, states).reshape(-1)

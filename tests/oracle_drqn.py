"""torch-CPU oracle of the DRQN update (xuance/torch/learners/qlearning_family/drqn_learner.py:12-80 on
DeepRecurrentQNetwork): float32 cuDNN-free nn.LSTM / nn.GRU, torch.optim.Adam (eps 1e-5) over the eval parameters,
clip_grad_norm_, LinearLR every update and a hard target sync every ``sync_frequency`` updates.  Parameter names are the
reference's, so its state_dict and the product's load into it with strict=True."""
from copy import deepcopy

import numpy as np
import torch
import torch.nn as nn


def seeded_state(template, seed):
    """A state_dict with the names and shapes of ``template`` (a DRQN network's), drawn from NumPy's PCG64 so that any
    machine rebuilds it bit for bit: eval matrices U(+-1/sqrt(fan_in)), biases U(+-0.1), and the target networks equal
    to the eval ones, as right after construction."""
    rng = np.random.default_rng(seed)
    out = {}
    for k, v in template.items():
        if k.startswith("target_"):
            continue
        shape = tuple(v.shape)
        scale = 1.0 / np.sqrt(shape[1]) if len(shape) == 2 else 0.1
        out[k] = torch.from_numpy((rng.uniform(-1.0, 1.0, shape) * scale).astype(np.float32))
    for k in template:
        if k.startswith("target_representation."):
            out[k] = out["representation." + k[len("target_representation."):]].clone()
        elif k.startswith("target_Q_head."):
            out[k] = out["eval_Q_head." + k[len("target_Q_head."):]].clone()
    return {k: out[k] for k in template}


class _Rep(nn.Module):
    def __init__(self, obs_dim, hidden):
        super().__init__()
        self.model = nn.Sequential(nn.Linear(obs_dim, hidden), nn.ReLU())


class _Head(nn.Module):
    def __init__(self, feat, H, A, rnn):
        super().__init__()
        self.lstm = rnn == "LSTM"
        self.rnn_layer = (nn.LSTM if self.lstm else nn.GRU)(feat, H, 1, batch_first=True)
        self.q_value = nn.Sequential(nn.Linear(H, A))

    def forward(self, x):
        y = self.rnn_layer(x)[0]
        return self.q_value(y)


class DRQNOracle(nn.Module):
    def __init__(self, rnn, H, obs_dim, rep_hidden, n_actions):
        super().__init__()
        self.representation = _Rep(obs_dim, rep_hidden)
        self.target_representation = deepcopy(self.representation)
        self.eval_Q_head = _Head(rep_hidden, H, n_actions, rnn)
        self.target_Q_head = deepcopy(self.eval_Q_head)

    def q(self, obs):
        return self.eval_Q_head(self.representation.model(obs))

    def target_q(self, obs):
        return self.target_Q_head(self.target_representation.model(obs))


class DRQNLearnerOracle:
    def __init__(self, model, lr=1e-3, gamma=0.99, sync_frequency=2, use_grad_clip=False, grad_clip_norm=0.5,
                 end_factor=0.5, total_iters=4):
        self.model, self.gamma, self.sync_frequency = model, gamma, sync_frequency
        self.use_grad_clip, self.grad_clip_norm = use_grad_clip, grad_clip_norm
        self.params = list(model.representation.parameters()) + list(model.eval_Q_head.parameters())
        self.optimizer = torch.optim.Adam(self.params, lr, eps=1e-5)
        self.scheduler = torch.optim.lr_scheduler.LinearLR(self.optimizer, 1.0, end_factor, total_iters)
        self.iterations = 0

    def update(self, obs, actions, rewards, terminals, **_):
        self.iterations += 1
        obs = torch.as_tensor(np.asarray(obs), dtype=torch.float32)
        act = torch.as_tensor(np.asarray(actions), dtype=torch.int64)
        rew = torch.as_tensor(np.asarray(rewards), dtype=torch.float32)
        ter = torch.as_tensor(np.asarray(terminals), dtype=torch.float32)
        evalQ = self.model.q(obs[:, :-1])
        with torch.no_grad():
            targetQ = self.model.target_q(obs[:, 1:]).max(dim=-1).values
        predictQ = evalQ.gather(-1, act.unsqueeze(-1)).squeeze(-1)
        y = rew + self.gamma * (1 - ter) * targetQ
        loss = ((predictQ - y) ** 2).mean()
        self.optimizer.zero_grad()
        loss.backward()
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(self.params, self.grad_clip_norm)
        self.optimizer.step()
        self.scheduler.step()
        if self.iterations % self.sync_frequency == 0:
            with torch.no_grad():
                for ep, tp in zip(self.model.representation.parameters(), self.model.target_representation.parameters()):
                    tp.copy_(ep)
                for ep, tp in zip(self.model.eval_Q_head.parameters(), self.model.target_Q_head.parameters()):
                    tp.copy_(ep)
        return {"Qloss": loss.item(), "learning_rate": self.optimizer.param_groups[0]["lr"],
                "predictQ": predictQ.mean().item()}

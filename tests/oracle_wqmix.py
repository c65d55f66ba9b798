"""Torch-CPU restatement of the reference Weighted QMIX update (OW-QMIX / CW-QMIX) for one parameter-sharing group with
GRU agents (use_rnn=True).  TEST INFRASTRUCTURE: the product never imports it.

  * QMIX_FF_Mixer ........................................ heads/q_mix_head.py:98-140
  * WeightedMixingQNetwork ............................... architectures/multi_agent/value_factorization.py:177-318
  * WQMIX_Learner._forward_transitions + update ........ learners/multi_agent_rl/wqmix_learner.py:27-227

``detach_q_eval=True`` is the reference as it runs: q_eval and q_eval_centralized are sliced inside torch.no_grad(), so
neither the agent networks nor the central agent networks receive a gradient and only the two mixers train.  ``False``
is the evidently intended computation (the slices outside no_grad).  The reference's double_q=False and CW-QMIX branches
raise as written (tests/golden/make_golden_wqmix.py); this restates them as intended: the unmasked argmax of the target
agent networks at t+1 without the extra axis, and ``batch.actions.group(group)``."""
import copy

import torch
import torch.nn as nn

from oracle.qmix import _AgentQ, MixerOracle


class FFMixerOracle(nn.Module):
    """q_mix_head.py:98-140."""

    def __init__(self, dim_state, dim_hidden, n_agents):
        super().__init__()
        self.S, self.n = dim_state, n_agents
        self.ff_net = nn.Sequential(nn.Linear(n_agents + dim_state, dim_hidden), nn.ReLU(),
                                    nn.Linear(dim_hidden, dim_hidden), nn.ReLU(),
                                    nn.Linear(dim_hidden, dim_hidden), nn.ReLU(), nn.Linear(dim_hidden, 1))
        self.ff_net_bias = nn.Sequential(nn.Linear(dim_state, dim_hidden), nn.ReLU(), nn.Linear(dim_hidden, 1))

    def forward(self, values_n, states):
        states = torch.as_tensor(states, dtype=torch.float32).reshape(-1, self.S)
        inputs = torch.cat([values_n.reshape(-1, self.n), states], dim=-1)
        return (self.ff_net(inputs) + self.ff_net_bias(states)).view(-1, 1)


class WQMIXModelOracle(nn.Module):
    def __init__(self, n_agents, obs_dim, n_actions, state_dim, hidden=64, mix_hidden=32, hyper_hidden=64,
                 ff_hidden=256):
        super().__init__()
        self.n_agents = n_agents
        self.individual_q_networks = nn.ModuleDict({'shared': _AgentQ(obs_dim, n_actions, hidden, hidden, (hidden,))})
        self.target_individual_q_networks = copy.deepcopy(self.individual_q_networks)
        self.eval_Qtot = MixerOracle(state_dim, mix_hidden, hyper_hidden, n_agents)
        self.target_Qtot = copy.deepcopy(self.eval_Qtot)
        self.individual_q_centralized = copy.deepcopy(self.individual_q_networks)
        self.target_individual_q_centralized = copy.deepcopy(self.individual_q_centralized)
        self.ff_mixer = FFMixerOracle(state_dim, ff_hidden, n_agents)
        self.target_ff_mixer = copy.deepcopy(self.ff_mixer)

    def parameters_model(self):
        return (list(self.individual_q_networks.parameters()) + list(self.eval_Qtot.parameters())
                + list(self.individual_q_centralized.parameters()) + list(self.ff_mixer.parameters()))

    def copy_target(self):
        for src, dst in ((self.individual_q_networks, self.target_individual_q_networks),
                         (self.eval_Qtot, self.target_Qtot),
                         (self.individual_q_centralized, self.target_individual_q_centralized),
                         (self.ff_mixer, self.target_ff_mixer)):
            for e, t in zip(src.parameters(), dst.parameters()):
                t.data.copy_(e)


class WQMIXLearnerOracle:
    def __init__(self, model, agent_keys, agent="OWQMIX", alpha=0.1, learning_rate=7e-4, gamma=0.99,
                 sync_frequency=200, double_q=True, use_grad_clip=False, grad_clip_norm=0.5, end_factor_lr_decay=1.0,
                 total_iters=1, detach_q_eval=True, use_actions_mask=True):
        assert agent in ("OWQMIX", "CWQMIX")
        self.model, self.agent_keys, self.agent, self.alpha = model, list(agent_keys), agent, alpha
        # LearnerMAS.build_optimizer (marl_learner.py:64-76): ONE Adam over model.parameters() (targets get no grads)
        self.optimizer = torch.optim.Adam(model.parameters(), lr=learning_rate, eps=1e-5, weight_decay=0.0)
        self.scheduler = torch.optim.lr_scheduler.LinearLR(self.optimizer, start_factor=1.0,
                                                           end_factor=end_factor_lr_decay, total_iters=total_iters)
        self.gamma, self.sync_frequency, self.double_q = gamma, sync_frequency, double_q
        self.use_grad_clip, self.grad_clip_norm = use_grad_clip, grad_clip_norm
        self.detach_q_eval, self.use_actions_mask = detach_q_eval, use_actions_mask
        self.iterations = 0

    def update(self, sample):
        self.iterations += 1
        K, B, T = self.agent_keys, sample['batch_size'], sample['sequence_length']
        n = len(K)
        st = lambda d, dt=None: torch.stack([torch.as_tensor(d[k], dtype=dt) for k in K], dim=1)
        obs, actions = st(sample['obs']), st(sample['actions'])               # [B, n, T+1, obs], [B, n, T]
        rewards, terminals = st(sample['rewards']), st(sample['terminals'], torch.float32)
        agent_mask = st(sample['agent_mask'], torch.float32)
        filled = torch.as_tensor(sample['filled'], dtype=torch.float32)        # [B, T]
        state = torch.as_tensor(sample['state'])                               # [B, T+1, S]
        avail = st(sample['avail_actions'], torch.float32) if self.use_actions_mask else None
        rewards_tot = rewards.mean(dim=1).reshape(-1)
        terminals_tot = (terminals != 0).all(dim=1).float().reshape(-1)
        m = self.model
        packed = obs.flatten(0, 1)
        q_all = m.individual_q_networks['shared'](packed).reshape(B, n, T + 1, -1)
        q_cent = m.individual_q_centralized['shared'](packed).reshape(B, n, T + 1, -1)
        with torch.no_grad():                                                  # value_factorization.py:87-92
            q_det = q_all.clone().detach()
            if avail is not None:
                q_det[avail == 0] = -1e10
            greedy = q_det.argmax(dim=-1)                                      # [B, n, T+1]
            q_next_cent = m.target_individual_q_centralized['shared'](packed).reshape(B, n, T + 1, -1)[:, :, 1:]
            if self.double_q:
                a_next = greedy[:, :, 1:]
            else:
                a_next = m.target_individual_q_networks['shared'](packed).reshape(B, n, T + 1, -1)[:, :, 1:].argmax(-1)
        q_eval, q_eval_cent = q_all[:, :, :-1], q_cent[:, :, :-1]
        if self.detach_q_eval:
            q_eval, q_eval_cent = q_eval.detach(), q_eval_cent.detach()
        g = greedy[:, :, :-1]
        mask = agent_mask * filled.unsqueeze(1).repeat(1, n, 1)               # valid_mask, outputs.py:133-143
        take = lambda q, idx: q.gather(-1, idx.long().unsqueeze(-1)).reshape(B, n, T)
        q_eval_taken = take(q_eval, actions) * mask
        q_cent_taken = take(q_eval_cent, g) * mask
        q_next_cent_taken = take(q_next_cent, a_next) * mask
        cat = lambda x: torch.concat([x[:, i].reshape(-1, 1) for i in range(n)], dim=-1)
        s_t, s_n = state[:, :-1].reshape(B * T, -1), state[:, 1:].reshape(B * T, -1)
        q_tot = m.eval_Qtot(cat(q_eval_taken), s_t).reshape(-1)
        q_ff = m.ff_mixer(cat(q_cent_taken), s_t).reshape(-1)
        with torch.no_grad():
            q_ff_next = m.target_ff_mixer(cat(q_next_cent_taken), s_n).reshape(-1)
        y = rewards_tot + (1 - terminals_tot) * self.gamma * q_ff_next
        td = q_tot - y.detach()
        ones = torch.ones_like(td)
        w = ones * self.alpha
        if self.agent == "CWQMIX":
            cond1 = ((g == actions) * mask).all(dim=1).reshape(-1)
            w = torch.where(cond1 | (y > q_ff), ones, w)
        else:
            w = torch.where(td < 0, ones, w)
        f = filled.reshape(-1)
        loss_central = (((q_ff - y.detach()) ** 2) * f).sum() / f.sum()
        loss_qmix = (w.detach() * (td ** 2) * f).sum() / f.sum()
        loss = loss_qmix + loss_central
        self.optimizer.zero_grad()
        loss.backward()
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(m.parameters(), self.grad_clip_norm)
        self.optimizer.step()
        self.scheduler.step()
        if self.iterations % self.sync_frequency == 0:
            m.copy_target()
        return {"learning_rate": self.optimizer.param_groups[0]['lr'], "loss_Qmix": loss_qmix.item(),
                "loss_central": loss_central.item(), "loss": loss.item(), "predictQ": q_tot.mean().item()}

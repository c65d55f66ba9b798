"""Torch-CPU restatement of the reference DCG / DCG_S update for one parameter-sharing group with GRU agents
(use_rnn=True).  TEST INFRASTRUCTURE: the product never imports it.

  * DCG_Utility, DCG_Payoff .............................. heads/coordination_graph.py:13-103
  * DeepCoordinationGraph ................................ architectures/multi_agent/value_factorization.py:450-590
  * DCG_Learner.act / q_dcg / _forward_transitions / update  learners/multi_agent_rl/dcg_learner.py:39-215

The greedy is the reference's float64 loop in its own summation orders (torch's mean, index_add_); K9C's documented
order can pick a different action only where two U values tie to within rounding (DESIGN.md section 4).  Parameter
names are the reference's, so the oracle, the product and a reference state_dict load into each other strictly."""
import copy

import torch
import torch.nn as nn


def reference_greedy(f, pay, edges, n_iter, normalize, avail):
    """dcg_learner.py:39-88 as the reference writes it (float64; torch's mean; scatter sums by index_add_, as the
    torch_scatter stub does): (actions [R, n], U [R, n, A]) from f [R, n, A] and raw payoffs [2, R, E, A*A]."""
    Rn, n, A = f.shape
    E = len(edges)
    fr = torch.tensor([e[0] for e in edges], dtype=torch.long)
    to = torch.tensor([e[1] for e in edges], dtype=torch.long)
    f_i = f.double() / n
    if E:
        P = pay.reshape(2, Rn, E, A, A).clone()
        P[1] = P[1].transpose(-1, -2).clone()
        f_ij = P.mean(dim=0).double() / E
        f_ji = f_ij.transpose(-1, -2).clone()
    scat = lambda src, idx: torch.zeros(Rn, n, A, dtype=src.dtype).index_add_(1, idx, src)
    m_ij = torch.zeros(Rn, E, A)
    m_ji = torch.zeros(Rn, E, A)
    U = f_i + scat(m_ij, to) + scat(m_ji, fr)
    if E:
        for _ in range(n_iter):
            jf = (U[:, fr, :] - m_ji).unsqueeze(-1) + f_ij
            jb = (U[:, to, :] - m_ij).unsqueeze(-1) + f_ji
            m_ij, m_ji = jf.max(dim=-2).values, jb.max(dim=-2).values
            if normalize:
                m_ij = m_ij - m_ij.mean(dim=-1, keepdim=True)
                m_ji = m_ji - m_ji.mean(dim=-1, keepdim=True)
            U = f_i + scat(m_ij, to) + scat(m_ji, fr)
    Um = U.clone()
    if avail is not None:
        Um[avail == 0] = -1e10
    return Um.argmax(dim=-1), U


class _RNNRep(nn.Module):
    def __init__(self, obs_dim, fc, hidden):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(obs_dim, fc), nn.ReLU())
        self.rnn = nn.GRU(fc, hidden, num_layers=1, batch_first=True)


class _Encoder(nn.Module):
    def __init__(self, obs_dim, fc, hidden):
        super().__init__()
        self.obs_representation = _RNNRep(obs_dim, fc, hidden)

    def forward(self, x):
        r = self.obs_representation
        return r.rnn(r.mlp(x))[0]


def _mlp(i, h, o):
    m = nn.Module()
    m.output = nn.Sequential(nn.Linear(i, h), nn.ReLU(), nn.Linear(h, o))
    return m


class DCGModelOracle(nn.Module):
    def __init__(self, n_agents, obs_dim, n_actions, state_dim=None, hidden=64, utility_hidden=64, payoff_hidden=64,
                 bias_hidden=64, low_rank=False, rank=1):
        super().__init__()
        self.n, self.A, self.low_rank, self.rank = n_agents, n_actions, low_rank, rank
        self.representation = nn.ModuleDict({'shared': _Encoder(obs_dim, hidden, hidden)})
        self.target_representation = copy.deepcopy(self.representation)
        self.utility = _mlp(hidden, utility_hidden, n_actions)
        self.target_utility = copy.deepcopy(self.utility)
        self.payoffs = _mlp(2 * hidden, payoff_hidden, 2 * rank * n_actions if low_rank else n_actions ** 2)
        self.target_payoffs = copy.deepcopy(self.payoffs)
        self.dcg_s = state_dim is not None
        if self.dcg_s:
            self.bias = nn.Module()
            self.bias.values = nn.Sequential(nn.Linear(state_dim, bias_hidden), nn.ReLU(), nn.Linear(bias_hidden, 1))
            self.target_bias = copy.deepcopy(self.bias)

    def raw_payoffs(self, h, edges, target=False):
        """h [R, n, H] -> raw payoff rows [2, R, E, A*A] (coordination_graph.py:90-101 before the symmetrisation)."""
        fr = torch.tensor([e[0] for e in edges], dtype=torch.long)
        to = torch.tensor([e[1] for e in edges], dtype=torch.long)
        x = torch.stack([torch.cat([h[:, fr], h[:, to]], dim=-1), torch.cat([h[:, to], h[:, fr]], dim=-1)], dim=0)
        out = (self.target_payoffs if target else self.payoffs).output(x)
        if not self.low_rank:
            return out
        lead, A = out.shape[:-1], self.A
        p = out.reshape(-1, 2, A)
        outer = torch.matmul(p[:, 0, :].unsqueeze(-1), p[:, 1, :].unsqueeze(-2))
        return outer.reshape(*lead, self.rank, A, A).sum(dim=-3).reshape(*lead, A * A)

    def copy_target(self):
        pairs = [(self.representation, self.target_representation), (self.utility, self.target_utility),
                 (self.payoffs, self.target_payoffs)]
        if self.dcg_s:
            pairs.append((self.bias, self.target_bias))
        for src, dst in pairs:
            for e, t in zip(src.parameters(), dst.parameters()):
                t.data.copy_(e)


class DCGLearnerOracle:
    def __init__(self, model, agent_keys, edges, n_msg_iterations=8, msg_normalized=True, learning_rate=7e-4,
                 gamma=0.99, sync_frequency=200, use_grad_clip=False, grad_clip_norm=0.5, end_factor_lr_decay=1.0,
                 total_iters=1, use_actions_mask=True):
        self.model, self.agent_keys, self.edges = model, list(agent_keys), list(edges)
        self.n_iter, self.normalize = n_msg_iterations, msg_normalized
        params = list(model.representation.parameters()) + list(model.utility.parameters()) + \
            list(model.payoffs.parameters()) + (list(model.bias.parameters()) if model.dcg_s else [])
        self.optimizer = torch.optim.Adam(params, lr=learning_rate, eps=1e-5)
        self.scheduler = torch.optim.lr_scheduler.LinearLR(self.optimizer, start_factor=1.0,
                                                           end_factor=end_factor_lr_decay, total_iters=total_iters)
        self.params = params
        self.gamma, self.sync_frequency = gamma, sync_frequency
        self.use_grad_clip, self.grad_clip_norm, self.use_actions_mask = use_grad_clip, grad_clip_norm, use_actions_mask
        self.iterations = 0

    def _q(self, h, acts, states, target):
        """q_dcg on h [R, n, H] with actions [R, n] (dcg_learner.py:90-104)."""
        m, E = self.model, len(self.edges)
        f = (m.target_utility if target else m.utility).output(h)
        A = f.shape[-1]
        q = (f.double() / m.n).gather(-1, acts.long().unsqueeze(-1)).sum(dim=1).squeeze(-1)
        if E > 0 and self.n_iter > 0:
            P = self.model.raw_payoffs(h, self.edges, target)
            fij = torch.stack([P[0].reshape(*P.shape[1:-1], A, A),
                               P[1].reshape(*P.shape[1:-1], A, A).transpose(-1, -2)]).mean(dim=0)
            fr = torch.tensor([e[0] for e in self.edges])
            to = torch.tensor([e[1] for e in self.edges])
            idx = (acts.long()[:, fr] * A + acts.long()[:, to]).unsqueeze(-1)
            q = q + (fij.double() / E).reshape(h.shape[0], E, A * A).gather(-1, idx).sum(dim=1).squeeze(-1)
        else:
            return q                                           # :95-96 returns before the DCG_S branch adds V(s)
        if m.dcg_s:
            q = q + m.bias.values(states).squeeze(-1)          # the ONLINE bias for both Q and Q' (:101)
        return q

    def greedy(self, h, avail=None):
        """act() on h [R, n, H] with the eval heads: the reference's float64 max-plus loop, in its summation orders."""
        with torch.no_grad():
            f = self.model.utility.output(h)
            pay = self.model.raw_payoffs(h, self.edges) if self.edges else None
        return reference_greedy(f, pay, self.edges, self.n_iter, self.normalize, avail)[0]

    def update(self, sample):
        self.iterations += 1
        K, B, T = self.agent_keys, sample['batch_size'], sample['sequence_length']
        n = len(K)
        st = lambda d, dt=None: torch.stack([torch.as_tensor(d[k], dtype=dt) for k in K], dim=1)
        obs, actions = st(sample['obs']), st(sample['actions'])               # [B, n, T+1, obs], [B, n, T]
        rewards, terminals = st(sample['rewards']), st(sample['terminals'], torch.float32)
        filled = torch.as_tensor(sample['filled'], dtype=torch.float32)        # [B, T]
        avail = st(sample['avail_actions'], torch.float32) if self.use_actions_mask else None
        m = self.model
        states = torch.as_tensor(sample['state'], dtype=torch.float32) if m.dcg_s else None
        rewards_tot = rewards.mean(dim=1).reshape(-1)
        terminals_tot = (terminals != 0).all(dim=1).float().reshape(-1)
        packed = obs.flatten(0, 1)
        h = m.representation['shared'](packed).reshape(B, n, T + 1, -1).transpose(1, 2)      # [B, T+1, n, H]
        with torch.no_grad():
            h_tgt = m.target_representation['shared'](packed).reshape(B, n, T + 1, -1).transpose(1, 2)
        rows = lambda x: x.reshape(B * T, *x.shape[2:])
        s_t = rows(states[:, :-1]) if states is not None else None
        s_n = rows(states[:, 1:]) if states is not None else None
        q_eval = self._q(rows(h[:, :-1]), rows(actions.transpose(1, 2)), s_t, False)
        av_next = rows(avail.transpose(1, 2)[:, 1:]) if avail is not None else None
        a_next = self.greedy(rows(h[:, 1:].detach()), av_next)
        with torch.no_grad():
            q_next = self._q(rows(h_tgt[:, 1:]), a_next, s_n, True)
        y = rewards_tot + (1 - terminals_tot) * self.gamma * q_next
        f = filled.reshape(-1)
        td = (q_eval - y.detach()) * f
        loss = (td ** 2).sum() / f.sum()
        self.optimizer.zero_grad()
        loss.backward()
        if self.use_grad_clip:
            torch.nn.utils.clip_grad_norm_(self.params, self.grad_clip_norm)
        self.optimizer.step()
        self.scheduler.step()
        if self.iterations % self.sync_frequency == 0:
            m.copy_target()
        return {"learning_rate": self.optimizer.param_groups[0]['lr'], "loss_Q": loss.item(),
                "predictQ": q_eval.mean().item()}

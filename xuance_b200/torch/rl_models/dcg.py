"""Deep Coordination Graph model pieces (reference: heads/coordination_graph.py:13-150,
architectures/multi_agent/value_factorization.py:450-590).  Module and parameter names mirror the reference so its
``state_dict`` loads with strict=True.  Scope: one parameter-sharing group of K13 GRU agents (use_rnn=True).

The utility and payoff MLPs are torch Linear layers (cuBLAS GEMMs).  Everything after them - the symmetrised payoff
f_ij = (P0 + P1^T) / 2, the max-plus message passing and the masked arg-max - is K9C (``xb_dcg_greedy``), which reads
the raw two-orientation payoff output, so the [.., E, A, A] f_ij tensor is never formed."""
from copy import deepcopy

import torch
import torch.nn as nn

from ... import _lib

MAX_AGENTS, MAX_ACTIONS, MAX_EDGES = 32, 64, 512   # K9C's limits (include/xb200.h)
MAX_SMEM = 227 * 1024


def greedy_smem_bytes(n, A, E):
    """Shared memory of one xb_dcg_greedy CTA: U [n, A] and both message sets [E, A] in float64, plus the edge list."""
    return 8 * (n * A + 2 * E * A) + 8 * E


def check_graph_limits(n, A, E):
    if n > MAX_AGENTS or A > MAX_ACTIONS or E > MAX_EDGES or greedy_smem_bytes(n, A, E) > MAX_SMEM:
        raise NotImplementedError(
            "DCG coordination-graph kernels: %d agents, %d actions and %d edges are outside the supported n <= %d, "
            "A <= %d, E <= %d with 8*(n*A + 2*E*A + E) <= %d bytes of shared memory"
            % (n, A, E, MAX_AGENTS, MAX_ACTIONS, MAX_EDGES, MAX_SMEM))


class DCG_Utility(nn.Module):
    """coordination_graph.py:13-48: Linear -> ReLU -> Linear, shared by every agent."""

    def __init__(self, dim_input, dim_hidden, dim_output, device=None):
        super().__init__()
        self.dim_input, self.dim_hidden, self.dim_output, self.device = dim_input, dim_hidden, dim_output, device
        self.output = nn.Sequential(nn.Linear(dim_input, dim_hidden), nn.ReLU(),
                                    nn.Linear(dim_hidden, dim_output)).to(device)

    def forward(self, hidden_states_n):
        return self.output(hidden_states_n)


class DCG_Payoff(DCG_Utility):
    """coordination_graph.py:51-103, without the symmetrisation (K9C does it): ``forward`` takes the stacked pair inputs
    [2, ..., 2H] and returns the raw payoff rows [2, ..., A*A].  With ``low_rank_payoff`` each output row is
    ``payoff_rank`` (u, v) pairs of A-vectors and the row is sum_k u_k v_k^T (a batched torch matmul)."""

    def __init__(self, dim_input, dim_hidden, dim_act, low_rank_payoff, payoff_rank, device=None):
        self.dim_act, self.low_rank_payoff, self.payoff_rank = dim_act, low_rank_payoff, payoff_rank
        dim_out = 2 * payoff_rank * dim_act if low_rank_payoff else dim_act ** 2
        super().__init__(dim_input, dim_hidden, dim_out, device)

    def forward(self, pair_inputs):
        out = self.output(pair_inputs)
        if not self.low_rank_payoff:
            return out
        lead, A = out.shape[:-1], self.dim_act
        f = out.reshape(-1, 2, A)                                     # [N*rank, 2, A], as coordination_graph.py:96
        outer = torch.matmul(f[:, 0, :].unsqueeze(-1), f[:, 1, :].unsqueeze(-2))
        return outer.reshape(*lead, self.payoff_rank, A, A).sum(dim=-3).reshape(*lead, A * A)


class Coordination_Graph:
    """coordination_graph.py:106-150: edge lists of the FULL, CYCLE, LINE, STAR and VDN (no edges) graphs, in the
    reference's order, as int32 device tensors."""

    def __init__(self, n_vertexes, graph_type="FULL", device=None):
        self.n_vertexes, self.device, self.graph_type = n_vertexes, device, graph_type
        n = n_vertexes
        if graph_type == "CYCLE":
            self.edges = [(i, i + 1) for i in range(n - 1)] + [(n - 1, 0)]
        elif graph_type == "LINE":
            self.edges = [(i, i + 1) for i in range(n - 1)]
        elif graph_type == "STAR":
            self.edges = [(0, i + 1) for i in range(n - 1)]
        elif graph_type == "VDN":
            self.edges = []
        elif graph_type == "FULL":
            self.edges = [(j, i + j + 1) for j in range(n - 1) for i in range(n - j - 1)]
        else:
            raise AttributeError("There is no graph type named {}!".format(graph_type))
        self.n_edges = len(self.edges)
        self.edges_from = self.edges_to = None

    def set_coordination_graph(self):
        self.edges_from = torch.tensor([e[0] for e in self.edges], dtype=torch.int32, device=self.device)
        self.edges_to = torch.tensor([e[1] for e in self.edges], dtype=torch.int32, device=self.device)


def pair_inputs(h, edges_from, edges_to):
    """h [B, n, T1, H] -> the payoff inputs [2, B, E, T1, 2H]: ([h_from, h_to], [h_to, h_from]) per edge."""
    hf, ht = h.index_select(1, edges_from), h.index_select(1, edges_to)
    return torch.stack([torch.cat([hf, ht], dim=-1), torch.cat([ht, hf], dim=-1)], dim=0)


def dcg_greedy(f, pay, graph, n_iter, normalize, T, t0, avail=None, U_out=None):
    """K9C greedy over f [B, n, T1, A] and pay [2, B, E, T1, A*A] (None when E = 0) at steps t0 .. t0+T-1 ->
    int32 actions [B*T, n].  avail [B, n, T1, A] uint8 or None; U_out [B*T, n, A] float64 or None."""
    B, n, T1, A = f.shape
    E = graph.n_edges
    actions = torch.empty((B * T, n), dtype=torch.int32, device=f.device)
    if avail is not None:
        assert avail.dtype == torch.uint8 and avail.is_contiguous() and tuple(avail.shape[:3]) == (B, n, T1)
    pay_ld = pay[0].numel() if pay is not None else 0
    _lib.call("xb_dcg_greedy", _lib.ptr(f), _lib.ptr(pay), pay_ld, _lib.ptr(graph.edges_from),
              _lib.ptr(graph.edges_to), _lib.ptr(avail), avail.shape[-1] if avail is not None else 0, B, T, T1, t0, n,
              A, E, int(n_iter), 1 if normalize else 0, _lib.ptr(actions), _lib.ptr(U_out))
    return actions


class DeepCoordinationGraph(nn.Module):
    """value_factorization.py:450-590 for one shared group: eval / target representation, utility, payoffs and (DCG_S)
    state-value bias.  ``forward`` is one acting step: a K13 GRU step, both heads and the K9C greedy."""

    def __init__(self, grouping, action_space, representation, utility, payoffs, dcg_graph, dcg_s=False, bias=None,
                 use_rnn=True, device=None, n_msg_iterations=8, msg_normalized=True, **kwargs):
        super().__init__()
        if not grouping.full_shared or not use_rnn:
            raise NotImplementedError("hot path scope: one parameter-sharing group with use_rnn=True")
        self.grouping, self.group_keys, self.agent_keys = grouping, grouping.group_keys, grouping.agent_keys
        self.action_space = action_space
        self.n_agents = len(self.agent_keys)
        self.dcg_s, self.use_rnn, self.device = dcg_s, use_rnn, device
        self.n_msg_iterations, self.msg_normalized = n_msg_iterations, msg_normalized
        self.dim_act = utility.dim_output
        check_graph_limits(self.n_agents, self.dim_act, dcg_graph.n_edges)
        self.representation = representation
        self.target_representation = deepcopy(representation)
        self.utility = utility
        self.target_utility = deepcopy(utility)
        self.payoffs = payoffs
        self.target_payoffs = deepcopy(payoffs)
        self.bias = bias
        self.target_bias = deepcopy(bias)
        self.graph = dcg_graph

    @property
    def parameters_model(self):
        params = list(self.representation.parameters()) + list(self.utility.parameters()) + \
            list(self.payoffs.parameters())
        if self.dcg_s:
            params += list(self.bias.parameters())
        return params

    @property
    def use_payoff(self):
        """q_dcg drops the payoff sum when the graph has no edges or no message passing runs (dcg_learner.py:95)."""
        return self.graph.n_edges > 0 and self.n_msg_iterations > 0

    def hidden_states(self, packed_obs, target=False):
        """packed_obs [B*n, T+1, obs] -> GRU outputs [B*n, T+1, H] from a zero initial state."""
        rep = (self.target_representation if target else self.representation)[self.group_keys[0]]
        return rep(packed_obs).embeddings

    def heads(self, h, target=False):
        """h [B, n, T1, H] -> (f [B, n, T1, A], pay [2, B, E, T1, A*A] or None when E = 0), contiguous."""
        utility = self.target_utility if target else self.utility
        payoffs = self.target_payoffs if target else self.payoffs
        f = utility(h).contiguous()
        if self.graph.n_edges == 0:
            return f, None
        pay = payoffs(pair_inputs(h, self.graph.edges_from, self.graph.edges_to)).contiguous()
        return f, pay

    def state_value(self, states, target=False):
        return (self.target_bias if target else self.bias)(states)

    # ---- acting: rows are (env, agent) pairs, agent-minor
    def init_rnn_states(self, n_envs):
        rep = self.representation[self.group_keys[0]].obs_representation
        return {self.group_keys[0]: rep.init_rnn_states(n_envs * self.n_agents)}

    def init_rnn_states_item(self, i_env, rnn_states):
        h = rnn_states[self.group_keys[0]]
        h[:, i_env * self.n_agents:(i_env + 1) * self.n_agents] = 0.0
        return rnn_states

    @torch.no_grad()
    def forward(self, observations, avail_actions=None, rnn_states=None, **kwargs):
        """observations [E*n, obs]; avail_actions [E*n, A] (non-zero = available) or None; rnn_states {group:
        [1, E*n, H]}.  Returns (greedy actions [E*n] int32, None, new rnn_states)."""
        g = self.group_keys[0]
        obs = torch.as_tensor(observations, dtype=torch.float32, device=self.device)
        h0 = None if rnn_states is None else rnn_states[g]
        rep = self.representation[g](obs, rnn_hidden=h0)
        h = rep.embeddings.reshape(-1, self.n_agents, 1, rep.embeddings.shape[-1])     # [E, n, 1, H]
        f, pay = self.heads(h)
        av = None
        if avail_actions is not None:
            av = (torch.as_tensor(avail_actions, device=self.device) != 0).to(torch.uint8)
            av = av.reshape(h.shape[0], self.n_agents, 1, -1).contiguous()
        actions = dcg_greedy(f, pay, self.graph, self.n_msg_iterations, self.msg_normalized, 1, 0, av)
        return actions.reshape(-1), None, {g: rep.rnn_states}

    def copy_target(self):
        for src, dst in ((self.representation, self.target_representation), (self.utility, self.target_utility),
                         (self.payoffs, self.target_payoffs)):
            for ep, tp in zip(src.parameters(), dst.parameters()):
                tp.data.copy_(ep)
        if self.dcg_s:
            for ep, tp in zip(self.bias.parameters(), self.target_bias.parameters()):
                tp.data.copy_(ep)

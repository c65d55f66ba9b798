"""QMIX model pieces (reference: representations/rnn.py:9-99, representations/agent_feature.py, critics/
base_critics.py:91-135, heads/q_mix_head.py:28-95, architectures/multi_agent/value_factorization.py:17-174).
Module / parameter names mirror the reference so its ``state_dict`` loads unchanged.  Scope: one parameter-sharing
group, GRU agents, discrete actions, no agent-identity encoding (mode 'none')."""
from copy import deepcopy

import torch
import torch.nn as nn

from ... import _lib
from .layers import mlp_block
from .heads import QValueHead
from .outputs import RepresentationOutput


class Basic_RNN(nn.Module):
    """rnn.py:9-99 (GRU variant): Linear+act stack -> GRU(batch_first)."""

    def __init__(self, input_shape, hidden_sizes=None, normalize=None, initialize=None, activation=None, device=None,
                 **kwargs):
        super().__init__()
        if kwargs.get("rnn", "GRU") != "GRU" or normalize is not None:
            raise NotImplementedError("only the un-normalised GRU variant is on the hot path")
        self.input_shape = input_shape
        self.fc_hidden_sizes = kwargs["fc_hidden_sizes"]
        self.recurrent_hidden_size = kwargs["recurrent_hidden_size"]
        self.N_recurrent_layer = kwargs.get("N_recurrent_layers", 1)
        self.device = device
        self.output_shapes = {'state': (self.recurrent_hidden_size,)}
        layers, shape = [], input_shape
        for h in self.fc_hidden_sizes:
            blk, shape = mlp_block(shape[0], h, None, activation, initialize, device=device)
            layers.extend(blk)
        self.mlp = nn.Sequential(*layers)
        self.rnn = nn.GRU(input_size=shape[0], hidden_size=self.recurrent_hidden_size,
                          num_layers=self.N_recurrent_layer, batch_first=True, dropout=kwargs.get("dropout", 0),
                          device=device)
        if initialize is not None:
            for wl in self.rnn.all_weights:
                for w in wl:
                    initialize(w) if len(w.shape) > 1 else nn.init.constant_(w, 0)

    def forward(self, x, rnn_hidden=None, **kwargs):
        x = torch.as_tensor(x, dtype=torch.float32, device=self.device)
        if rnn_hidden is None:
            rnn_hidden = self.init_rnn_states(x.shape[0])
        out, hn = self.rnn(self.mlp(x), rnn_hidden)
        return RepresentationOutput(embeddings=out, rnn_states=hn.detach())

    def init_rnn_states(self, batch):
        return torch.zeros((self.N_recurrent_layer, batch, self.recurrent_hidden_size), device=self.device)


class AgentFeatureEncoder(nn.Module):
    """agent_feature.py with identity mode 'none': passes the observation representation through."""

    def __init__(self, representation):
        super().__init__()
        self.obs_representation = representation
        self.output_shapes = representation.output_shapes

    def forward(self, observations, **kwargs):
        return self.obs_representation(observations, **kwargs)


class DiscreteActionValueCritic(nn.Module):
    """base_critics.py:91-135."""

    def __init__(self, representation, action_space, critic_hidden_size, normalizer=None, initializer=None,
                 activation=None, device=None, **kwargs):
        super().__init__()
        self.action_space, self.n_actions = action_space, action_space.n
        self.representation = representation
        self.critic_head = QValueHead(feature_dim=representation.output_shapes['state'][0],
                                      hidden_size=critic_hidden_size, n_actions=self.n_actions, normalizer=normalizer,
                                      initializer=initializer, activation=activation, device=device)

    def forward(self, observation, **kwargs):
        rep = self.representation(observation, **kwargs)
        return self.critic_head(rep.embeddings), rep


class _MixFunction(torch.autograd.Function):
    """hidden = elu(q.|w1| + b1); q_tot = hidden.|w2| + b2 per row - K9 mix forward / backward."""

    @staticmethod
    def forward(ctx, q, w1, b1, w2, b2, n, H):
        q, w1, b1, w2, b2 = (x.contiguous() for x in (q, w1, b1, w2, b2))
        R = q.shape[0]
        out = torch.empty(R, dtype=torch.float32, device=q.device)
        _lib.call("xb_qmix_mix_fwd", _lib.ptr(q), _lib.ptr(w1), _lib.ptr(b1), _lib.ptr(w2), _lib.ptr(b2), R, n, H,
                  _lib.ptr(out))
        ctx.save_for_backward(q, w1, b1, w2)
        ctx.dims = (n, H)
        return out

    @staticmethod
    def backward(ctx, dy):
        q, w1, b1, w2 = ctx.saved_tensors
        n, H = ctx.dims
        dy = dy.contiguous()
        R = q.shape[0]
        dq, dw1 = torch.empty_like(q), torch.empty_like(w1)
        db1, dw2 = torch.empty_like(b1), torch.empty_like(w2)
        _lib.call("xb_qmix_mix_bwd", _lib.ptr(dy), _lib.ptr(q), _lib.ptr(w1), _lib.ptr(b1), _lib.ptr(w2), R, n, H,
                  _lib.ptr(dq), _lib.ptr(dw1), _lib.ptr(db1), _lib.ptr(dw2))
        return dq, dw1, db1, dw2, dy, None, None


class QMIX_Mixer(nn.Module):
    """q_mix_head.py:28-95.  The four hypernetworks are torch Linear layers (cuBLAS GEMMs); everything after them
    - abs, the two per-row contractions, ELU, bias - is one fused K9 launch in each direction."""

    def __init__(self, dim_state=None, dim_hidden=32, dim_hypernet_hidden=32, n_agents=1, device=None):
        super().__init__()
        self.device, self.dim_state, self.dim_hidden = device, dim_state, dim_hidden
        self.dim_hypernet_hidden, self.n_agents = dim_hypernet_hidden, n_agents
        self.hyper_w_1 = nn.Sequential(nn.Linear(dim_state, dim_hypernet_hidden), nn.ReLU(),
                                       nn.Linear(dim_hypernet_hidden, dim_hidden * n_agents)).to(device)
        self.hyper_w_2 = nn.Sequential(nn.Linear(dim_state, dim_hypernet_hidden), nn.ReLU(),
                                       nn.Linear(dim_hypernet_hidden, dim_hidden)).to(device)
        self.hyper_b_1 = nn.Linear(dim_state, dim_hidden).to(device)
        self.hyper_b_2 = nn.Sequential(nn.Linear(dim_state, dim_hypernet_hidden), nn.ReLU(),
                                       nn.Linear(dim_hypernet_hidden, 1)).to(device)

    use_tensor_core_forward = True   # no-grad forwards (target mixer, inference) take the fused wgmma kernel

    def _fusable(self):
        kp1 = (self.dim_state + 15) // 16 * 16
        smem = 1024 * kp1 + 4096 * self.n_agents + 6144 + 512 * self.dim_state   # operands + raw X tile of K9-TC (bytes)
        return (self.use_tensor_core_forward and self.dim_hidden == 32 and self.dim_hypernet_hidden == 32
                and self.n_agents <= 8 and smem <= 220 * 1024 and kp1 >= 96)

    def forward_fused(self, values_n, states):
        """Whole mixer in ONE tensor-core kernel (K9-TC, xb_qmix_mix_fused_fwd).  Forward only."""
        states = torch.as_tensor(states, dtype=torch.float32, device=self.device).reshape(-1, self.dim_state).contiguous()
        q = values_n.reshape(-1, self.n_agents).to(torch.float32).contiguous()
        import ctypes
        l1 = [self.hyper_w_1[0], self.hyper_b_1, self.hyper_w_2[0], self.hyper_b_2[0]]
        w_ptrs = (ctypes.c_void_p * 4)(*[_lib.ptr(m.weight.contiguous()) for m in l1])
        b_ptrs = (ctypes.c_void_p * 4)(*[_lib.ptr(m.bias.contiguous()) for m in l1])
        R = q.shape[0]
        out = torch.empty(R, dtype=torch.float32, device=q.device)
        l2 = [self.hyper_w_1[2].weight, self.hyper_w_1[2].bias, self.hyper_w_2[2].weight, self.hyper_w_2[2].bias,
              self.hyper_b_2[2].weight, self.hyper_b_2[2].bias]
        _lib.call("xb_qmix_mix_fused_fwd", _lib.ptr(states), _lib.ptr(q), w_ptrs, b_ptrs,
                  *[_lib.ptr(t.contiguous()) for t in l2], R, self.dim_state, self.n_agents, self.dim_hidden,
                  self.dim_hypernet_hidden, _lib.ptr(out))
        return out.view(-1, 1)

    def forward(self, values_n, states):
        if not torch.is_grad_enabled() and self._fusable():
            return self.forward_fused(values_n, states)
        states = torch.as_tensor(states, dtype=torch.float32, device=self.device).reshape(-1, self.dim_state)
        q = values_n.reshape(-1, self.n_agents)
        w1 = self.hyper_w_1(states)          # abs() is applied inside the fused kernel
        b1 = self.hyper_b_1(states)
        w2 = self.hyper_w_2(states)
        b2 = self.hyper_b_2(states).reshape(-1)
        return _MixFunction.apply(q, w1, b1, w2, b2, self.n_agents, self.dim_hidden).view(-1, 1)


class QMIX_FF_Mixer(nn.Module):
    """q_mix_head.py:98-140: the unconstrained feed-forward mixer of Weighted QMIX,
    q_tot = ff_net([q, s]) + ff_net_bias(s).  Its layers are torch Linear layers (cuBLAS GEMMs) with torch's default
    initialisation, as in the reference."""

    def __init__(self, dim_state=0, dim_hidden=32, n_agents=1, device=None):
        super().__init__()
        self.device, self.dim_state, self.dim_hidden, self.n_agents = device, dim_state, dim_hidden, n_agents
        self.dim_input = n_agents + dim_state
        self.ff_net = nn.Sequential(nn.Linear(self.dim_input, dim_hidden), nn.ReLU(),
                                    nn.Linear(dim_hidden, dim_hidden), nn.ReLU(),
                                    nn.Linear(dim_hidden, dim_hidden), nn.ReLU(),
                                    nn.Linear(dim_hidden, 1)).to(device)
        self.ff_net_bias = nn.Sequential(nn.Linear(dim_state, dim_hidden), nn.ReLU(),
                                         nn.Linear(dim_hidden, 1)).to(device)

    def forward(self, values_n, states=None):
        states = torch.as_tensor(states, dtype=torch.float32, device=self.device).reshape(-1, self.dim_state)
        inputs = torch.cat([values_n.reshape(-1, self.n_agents), states], dim=-1)
        return (self.ff_net(inputs) + self.ff_net_bias(states)).view(-1, 1)


class VDN_mixer(nn.Module):
    """q_mix_head.py VDN_mixer: Q_tot = sum_i Q_i (no parameters, the global state is ignored)."""

    def __init__(self, *args, **kwargs):
        super().__init__()

    def forward(self, values_n, states=None):
        return values_n.reshape(values_n.shape[0] if values_n.dim() == 2 else -1, -1).sum(dim=-1, keepdim=True)


class IndependentMixer(nn.Module):
    """q_mix_head.py IndependentMixer: independent Q-learning, the agents' values pass through (no parameters).  IQL's
    update never calls it: its loss is per agent (K9I)."""

    def forward(self, values_n, states=None):
        return values_n


class MixingQNetwork(nn.Module):
    """value_factorization.py:17-174 for one shared group: eval/target agent networks + eval/target mixers."""

    def __init__(self, grouping, q_networks, mixer, use_rnn=True, device=None, **kwargs):
        super().__init__()
        if not grouping.full_shared or not use_rnn:
            raise NotImplementedError("hot path scope: one parameter-sharing group with use_rnn=True")
        self.grouping, self.group_keys, self.agent_keys = grouping, grouping.group_keys, grouping.agent_keys
        self.n_agents = len(self.agent_keys)
        self.use_rnn, self.device = use_rnn, device
        self.individual_q_networks = q_networks
        self.target_individual_q_networks = deepcopy(q_networks)
        self.eval_Qtot = mixer
        self.target_Qtot = deepcopy(mixer)

    @property
    def parameters_model(self):
        return list(self.individual_q_networks.parameters()) + list(self.eval_Qtot.parameters())

    def q_values(self, packed_obs, target=False):
        """packed_obs [B*n, T+1, obs] -> Q [B*n, T+1, A] (GRU from a zero initial state, as init_rnn_states)."""
        net = (self.target_individual_q_networks if target else self.individual_q_networks)[self.group_keys[0]]
        return net(packed_obs)[0]

    # ---- acting (value_factorization.py:54-96 for one time step): rows are (env, agent) pairs, agent-minor
    def init_rnn_states(self, n_envs):
        rep = self.individual_q_networks[self.group_keys[0]].representation.obs_representation
        return {self.group_keys[0]: rep.init_rnn_states(n_envs * self.n_agents)}

    def init_rnn_states_item(self, i_env, rnn_states):
        h = rnn_states[self.group_keys[0]]
        h[:, i_env * self.n_agents:(i_env + 1) * self.n_agents] = 0.0
        return rnn_states

    @torch.no_grad()
    def forward(self, observations, avail_actions=None, rnn_states=None, **kwargs):
        """observations [E*n, 1, obs] (or [E*n, obs]); avail_actions [E*n, A] (non-zero = available) or None;
        rnn_states {group: [layers, E*n, H]}.  Returns (greedy actions [E*n] int64, q [E*n, A], new rnn_states): the
        arg-max runs over q with unavailable actions at -1e10 (value_factorization.py:86-91)."""
        g = self.group_keys[0]
        obs = torch.as_tensor(observations, dtype=torch.float32, device=self.device)
        if obs.dim() == 2:
            obs = obs.unsqueeze(1)
        h0 = None if rnn_states is None else rnn_states[g]
        q, rep = self.individual_q_networks[g](obs, rnn_hidden=h0)
        q = q[:, -1]
        q_sel = q
        if avail_actions is not None:
            av = torch.as_tensor(avail_actions, device=self.device)
            q_sel = q.masked_fill(av == 0, -1e10)
        return q_sel.argmax(dim=-1), q, {g: rep.rnn_states}

    def Q_tot(self, q_taken, states):
        return self.eval_Qtot(q_taken, states)

    def Qtarget_tot(self, q_taken, states):
        return self.target_Qtot(q_taken, states)

    def copy_target(self):
        for ep, tp in zip(self.individual_q_networks.parameters(), self.target_individual_q_networks.parameters()):
            tp.data.copy_(ep)
        for ep, tp in zip(self.eval_Qtot.parameters(), self.target_Qtot.parameters()):
            tp.data.copy_(ep)


class WeightedMixingQNetwork(MixingQNetwork):
    """value_factorization.py:177-318: MixingQNetwork plus the central agent networks (a deep copy of the agent networks,
    own GRU, on cuDNN like them), the feed-forward mixer and a target copy of each.  Submodules are registered in the
    reference's order, so its state_dict loads strictly."""

    def __init__(self, grouping, q_networks, mixer, ff_mixer, use_rnn=True, device=None, **kwargs):
        super().__init__(grouping, q_networks, mixer, use_rnn=use_rnn, device=device, **kwargs)
        self.individual_q_centralized = deepcopy(q_networks)
        self.target_individual_q_centralized = deepcopy(self.individual_q_centralized)
        self.ff_mixer = ff_mixer
        self.target_ff_mixer = deepcopy(ff_mixer)

    @property
    def parameters_model(self):
        return (list(self.individual_q_networks.parameters()) + list(self.eval_Qtot.parameters())
                + list(self.individual_q_centralized.parameters()) + list(self.ff_mixer.parameters()))

    def q_centralized(self, packed_obs, target=False):
        """packed_obs [B*n, T+1, obs] -> central Q [B*n, T+1, A] from a zero initial state."""
        nets = self.target_individual_q_centralized if target else self.individual_q_centralized
        return nets[self.group_keys[0]](packed_obs)[0]

    def q_feedforward(self, q_taken, states):
        return self.ff_mixer(q_taken, states)

    def target_q_feedforward(self, q_taken, states):
        return self.target_ff_mixer(q_taken, states)

    def copy_target(self):
        super().copy_target()
        for ep, tp in zip(self.individual_q_centralized.parameters(), self.target_individual_q_centralized.parameters()):
            tp.data.copy_(ep)
        for ep, tp in zip(self.ff_mixer.parameters(), self.target_ff_mixer.parameters()):
            tp.data.copy_(ep)

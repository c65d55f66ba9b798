"""Episode replay for recurrent off-policy MARL (QMIX) - mirror of MARL_OffPolicyBuffer_RNN
(xuance/common/memory_tools_marl.py:770-996).

Same ``store(**step_data) / finish_path(i_env, **terminal_data) / sample()`` surface and sample-dict keys.  The
per-env episode scratch (``episode_data``) stays on the host - it is written a few hundred bytes at a time by the
vector env loop - while the replay ring (``data``) lives in HBM, agent-stacked ``[capacity, n_agents, T(+1), dim]``
so that one K1 row-store per field ingests a finished episode and one K3 row-gather per field builds a batch
already in the ``[B, n_agents, T(+1), dim]`` layout the learner consumes (the reference re-stacks per-agent
dicts on every update, marl_learner.py:336-394).  ``sample()`` returns per-agent views of those stacked tensors
under the reference's keys, plus the stacked tensors themselves under ``'_stacked'``.

``MARL_OnPolicyBuffer`` mirrors memory_tools_marl.py:63-270 for feed-forward MAPPO (see its docstring)."""
import numpy as np
import torch

from .. import _lib
from .spaces import space2shape


def _pad4(n):
    return (n + 3) // 4 * 4


class _MARLBuffer:
    """The construction every multi-agent buffer shares: one parameter-sharing group (all agents with the same
    observation and action shapes), Discrete actions (each subclass refuses a Box with its ``BOX_REFUSAL``) and
    storage on a CUDA device."""
    BOX_REFUSAL = None

    def __init__(self, agent_keys, state_space, obs_space, act_space, n_envs, buffer_size, device, **kwargs):
        self.agent_keys = list(agent_keys)
        self.n_agents = len(self.agent_keys)
        self.n_envs, self.buffer_size = n_envs, buffer_size
        self.state_space = state_space
        self.store_global_state = state_space is not None
        self.use_actions_mask = kwargs.get("use_actions_mask", False)
        self.avail_actions_shape = kwargs.get("avail_actions_shape", None)
        self.obs_shape = {k: tuple(space2shape(obs_space[k])) for k in self.agent_keys}
        self.act_shape = {k: tuple(space2shape(act_space[k])) for k in self.agent_keys}
        k0 = self.agent_keys[0]
        if any(self.obs_shape[k] != self.obs_shape[k0] or self.act_shape[k] != self.act_shape[k0] for k in self.agent_keys):
            raise NotImplementedError("heterogeneous agents are outside the hot-path scope (one parameter-sharing group)")
        if self.act_shape[k0] != ():
            raise NotImplementedError(self.BOX_REFUSAL)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("xuance_b200 buffers are device-resident: device must be CUDA (no CPU fallback)")
        _lib.load()
        _lib.use_device(self.device)
        self._obs_dim = int(np.prod(self.obs_shape[k0]))
        self._state_dim = int(np.prod(space2shape(state_space))) if self.store_global_state else 0
        self._n_act = int(self.avail_actions_shape[k0][0]) if self.use_actions_mask else 0

    def _gather_rows(self, src, idx_t):
        """K3: src[idx_t] for rows of src.shape[1:]."""
        out = torch.empty((idx_t.numel(),) + tuple(src.shape[1:]), dtype=src.dtype, device=self.device)
        row_bytes = int(np.prod(src.shape[1:])) * src.element_size()
        _lib.call("xb_gather_rows", _lib.ptr(src), _lib.ptr(idx_t), idx_t.numel(), row_bytes, _lib.ptr(out))
        return out


class _MARLOnPolicyBuffer(_MARLBuffer):
    """What the two on-policy buffers share: the scalar fields, the (env, agent) rows, the GAE launch and the per-agent
    split of a sample."""
    FIELDS = ('actions', 'rewards', 'values', 'log_pi_old', 'terminals', 'agent_mask', 'returns', 'advantages')
    STORED = 6   # the fields store() writes; returns / advantages come from finish_path

    def __init__(self, agent_keys, state_space, obs_space, act_space, n_envs, buffer_size, use_gae, use_advnorm, gamma,
                 gae_lam, device, **kwargs):
        super().__init__(agent_keys, state_space, obs_space, act_space, n_envs, buffer_size, device, **kwargs)
        self.use_gae, self.use_advantage_norm = use_gae, use_advnorm
        self.gamma, self.gae_lambda = gamma, gae_lam
        self._rows = self.n_envs * self.n_agents

    def _per_agent(self, d, dtype=np.float32):
        """{agent: [n_envs, ...]} -> [n_envs * n_agents, ...] (env-major, agent-minor)."""
        return np.stack([np.asarray(d[k], dtype=dtype) for k in self.agent_keys], axis=1).reshape(self._rows, -1)

    def _gae(self, rows, seg_end, boot, start, cov, agent_grouping, value_normalizer):
        """``xb_gae_scan_vn`` over the agent rows ``rows`` of ``field()``: advantages and returns of the path that ends
        where ``seg_end`` marks it (bootstrapping from ``boot``), on the steps [start, cov) of each row (start None: 0),
        with the values denormalised by the group's ValueNorm state as it is now."""
        vn = None
        if value_normalizer is not None:
            groups = {agent_grouping.agent_to_group[k] for k in self.agent_keys} if agent_grouping is not None \
                else set(value_normalizer)
            if len(groups) != 1:
                raise NotImplementedError("one parameter-sharing group")
            vn = value_normalizer[groups.pop()]
        vp = vn.state_pointers() if vn is not None else (None, None, None)
        f = lambda name: _lib.ptr(self.field(name)[rows])
        _lib.call("xb_gae_scan_vn", f('rewards'), f('values'), f('terminals'), _lib.ptr(seg_end), _lib.ptr(boot),
                  _lib.ptr(start), _lib.ptr(cov), f('advantages'), f('returns'), self.n_agents,
                  self.field('rewards').shape[1], float(self.gamma),
                  float(self.gae_lambda if self.gae_lambda is not None else 0.0), 1 if self.use_gae else 0, *vp)

    def _split(self, st, B):
        """The agent-major stacked sample (row k * B + b is agent k of sample b) as per-agent views under the
        reference's keys; the per-sample ``filled`` and ``state`` keep agent 0's rows."""
        out = {}
        for key, v in st.items():
            if key == 'avail_actions':
                v = v[..., :self._n_act]
            if key in ('terminals', 'agent_mask', 'avail_actions', 'filled'):
                v = v.bool()
            out[key] = v[:B] if key in ('filled', 'state') else {a: v[i * B:(i + 1) * B]
                                                                 for i, a in enumerate(self.agent_keys)}
        return out


class MARL_OffPolicyBuffer_RNN(_MARLBuffer):
    BOX_REFUSAL = "QMIX uses discrete actions"

    def __init__(self, agent_keys, state_space=None, obs_space=None, act_space=None, n_envs=1, buffer_size=1,
                 batch_size=1, max_episode_steps=1, device="cuda:0", **kwargs):
        assert buffer_size % n_envs == 0, "buffer_size must be divisible by the number of envs (parallels)"
        super().__init__(agent_keys, state_space, obs_space, act_space, n_envs, buffer_size, device, **kwargs)
        self.batch_size, self.max_eps_len = batch_size, max_episode_steps
        self.clear()
        self.clear_episodes()

    # ---- field table: name -> (per-episode shape, dtype, per-agent?)
    def _fields(self):
        n, T, Tp = self.n_agents, self.max_eps_len, _pad4(self.max_eps_len)
        f = {'obs': ((n, T + 1, self._obs_dim), torch.float32), 'actions': ((n, T), torch.float32),
             'rewards': ((n, T), torch.float32), 'terminals': ((n, Tp), torch.uint8),
             'agent_mask': ((n, Tp), torch.uint8), 'filled': ((Tp,), torch.uint8)}
        if self.store_global_state:
            f['state'] = ((T + 1, self._state_dim), torch.float32)
        if self.use_actions_mask:
            f['avail_actions'] = ((n, T + 1, _pad4(self._n_act)), torch.uint8)
        return f

    @property
    def data_keys(self):
        return list(self._fields().keys())

    def clear(self):
        self._dev = {k: torch.zeros((self.buffer_size,) + s, dtype=dt, device=self.device)
                     for k, (s, dt) in self._fields().items()}
        self.ptr, self.size = 0, 0

    def clear_episodes(self):
        self.episode_data = {k: torch.zeros((self.n_envs,) + s, dtype=dt).pin_memory()
                             for k, (s, dt) in self._fields().items()}
        self._ep_np = {k: v.numpy() for k, v in self.episode_data.items()}

    # ---- checkpoint (SURVEY.md section 8f-4; the reference does not save its replay)
    def state_dict(self):
        return {"class": type(self).__name__, "buffer_size": self.buffer_size, "n_envs": self.n_envs,
                "max_eps_len": self.max_eps_len, "ptr": int(self.ptr), "size": int(self.size),
                "data": {k: v.cpu() for k, v in self._dev.items()},
                "episode_data": {k: v.clone() for k, v in self.episode_data.items()}}

    def load_state_dict(self, sd):
        if (sd.get("class"), sd.get("buffer_size"), sd.get("n_envs"), sd.get("max_eps_len")) != \
                (type(self).__name__, self.buffer_size, self.n_envs, self.max_eps_len):
            raise ValueError("episode-replay checkpoint does not match this buffer's capacity / envs / episode length")
        for k, v in self._dev.items():
            if tuple(sd["data"][k].shape) != tuple(v.shape) or sd["data"][k].dtype != v.dtype:
                raise ValueError("episode-replay checkpoint field %s has shape %s" % (k, tuple(sd["data"][k].shape)))
            v.copy_(sd["data"][k])
        for k, v in self.episode_data.items():
            v.copy_(sd["episode_data"][k])
        self.ptr, self.size = int(sd["ptr"]), int(sd["size"])

    @property
    def full(self):
        return self.size >= self.buffer_size

    def can_sample(self):
        return self.size >= self.batch_size

    # ---- reference :912-929
    def store(self, **step_data):
        steps = step_data['episode_steps']
        envs = np.arange(self.n_envs)
        ep = self._ep_np
        ep['filled'][envs, steps] = 1
        for key, val in step_data.items():
            if key not in ep or key == 'filled':
                continue
            if key == 'state':
                ep['state'][envs, steps] = val
                continue
            for i, a in enumerate(self.agent_keys):
                if key == 'avail_actions':
                    ep[key][envs, i, steps, :self._n_act] = val[a]
                else:
                    ep[key][envs, i, steps] = val[a]

    # ---- reference :952-969 (+ store_episodes :931-950): terminal obs/state, then the episode goes to HBM
    def finish_path(self, i_env, **terminal_data):
        t = terminal_data['episode_step']
        ep = self._ep_np
        if self.store_global_state:
            ep['state'][i_env, t] = terminal_data['state']
        for i, a in enumerate(self.agent_keys):
            ep['obs'][i_env, i, t] = terminal_data['obs'][a]
            if self.use_actions_mask:
                ep['avail_actions'][i_env, i, t, :self._n_act] = terminal_data['avail_actions'][a]
        for key, dst in self._dev.items():
            row = self.episode_data[key][i_env:i_env + 1].to(self.device, non_blocking=True)
            flat = row.reshape(1, -1)
            row_bytes = flat.shape[1] * flat.element_size()
            # K1 rows path with N=1 "env", T=capacity slots: dst[0, ptr] = row
            _lib.call("xb_rollout_store", _lib.ptr(dst), _lib.ptr(flat), row_bytes, None, None, 0, 1,
                      self.buffer_size, int(self.ptr))
        torch.cuda.current_stream().synchronize()   # the pinned scratch row is reused right away
        self.ptr = (self.ptr + 1) % self.buffer_size
        self.size = min(self.size + 1, self.buffer_size)
        ep['filled'][i_env] = 0

    # ---- reference :971-996
    def sample(self, batch_size=None, episode_choices=None):
        assert self.size > 0, "You need to first store experience data into the buffer!"
        if batch_size is None:
            batch_size = self.batch_size
        if episode_choices is None:
            episode_choices = np.random.choice(self.size, batch_size)
        idx_t = torch.from_numpy(np.asarray(episode_choices, dtype=np.int64)).to(self.device)
        T, A = self.max_eps_len, self._n_act
        st = {k: self._gather_rows(v, idx_t) for k, v in self._dev.items()}
        st['terminals'] = st['terminals'][:, :, :T].bool()
        st['agent_mask'] = st['agent_mask'][:, :, :T].bool()
        st['filled'] = st['filled'][:, :T].bool()
        if self.use_actions_mask:
            st['avail_actions'] = st['avail_actions'][..., :A].bool()
        out = {}
        for key, v in st.items():
            out[key] = v if key in ('filled', 'state') else {a: v[:, i] for i, a in enumerate(self.agent_keys)}
        out['batch_size'] = batch_size
        out['sequence_length'] = T
        out['_stacked'] = st
        return out


class MARL_OnPolicyBuffer(_MARLOnPolicyBuffer):
    """On-policy multi-agent rollout - mirror of MARL_OnPolicyBuffer (xuance/common/memory_tools_marl.py:63-270):
    ``store(**step_data)``, ``finish_path(i_env, agent_grouping, value_next, value_normalizer)``, ``sample(indexes)``,
    ``clear``, ``full``, ``ptr / size / start_ids``, same constructor arguments and sample keys.

    The rollout lives in HBM.  Rows are (env, agent) pairs, row = env * n_agents + agent, so the scalar fields
    ``[F, n_envs * n_agents, n_size]`` are K2's layout with the agents as extra envs, and one K1 launch stores a vector
    step.  ``finish_path`` runs ``xb_gae_scan_vn`` over the finished env's rows at once, denormalising with the
    ValueNorm state as it is at that moment (the reference's per-step Python loop, :208-236).  ``sample`` gathers the
    minibatch agent-major (row k * B + b is agent k of sample b) with K3 and normalises the advantages per agent over
    the minibatch, as the reference does per agent key (:255-258)."""
    BOX_REFUSAL = "MARL_OnPolicyBuffer: Box action spaces (Gaussian MAPPO) are not supported"

    def __init__(self, agent_keys, state_space=None, obs_space=None, act_space=None, n_envs=1, buffer_size=1,
                 use_gae=False, use_advnorm=False, gamma=None, gae_lam=None, device="cuda:0", **kwargs):
        assert buffer_size % n_envs == 0, "buffer_size must be divisible by the number of envs (parallels)"
        super().__init__(agent_keys, state_space, obs_space, act_space, n_envs, buffer_size, use_gae, use_advnorm,
                         gamma, gae_lam, device, **kwargs)
        self.n_size = buffer_size // n_envs
        self._scratch = _lib.scratch(self.device)
        self.clear()

    @property
    def data_keys(self):
        keys = ['obs'] + list(self.FIELDS)
        if self.store_global_state:
            keys.append('state')
        if self.use_actions_mask:
            keys.append('avail_actions')
        return keys

    @property
    def full(self):
        return self.size >= self.n_size

    def clear(self):
        R, T, dev = self._rows, self.n_size, self.device
        self._scal = torch.zeros((len(self.FIELDS), R, T), dtype=torch.float32, device=dev)
        self._obs = torch.zeros((R, T, self._obs_dim), dtype=torch.float32, device=dev)
        self._avail = (torch.zeros((R, T, _pad4(self._n_act)), dtype=torch.uint8, device=dev)
                       if self.use_actions_mask else None)
        self._state = (torch.zeros((self.n_envs, T, self._state_dim), dtype=torch.float32, device=dev)
                       if self.store_global_state else None)
        self._seg_end = np.zeros((R, T), np.uint8)
        self._boot = np.zeros((R, T), np.float32)
        self._seg_end_d = torch.zeros((R, T), dtype=torch.uint8, device=dev)
        self._boot_d = torch.zeros((R, T), dtype=torch.float32, device=dev)
        self._start_d = torch.zeros(R, dtype=torch.int32, device=dev)
        self._cov_d = torch.zeros(R, dtype=torch.int32, device=dev)
        self.ptr, self.size = 0, 0
        self.start_ids = np.zeros(self.n_envs, np.int64)

    def field(self, name):
        """[n_envs * n_agents, n_size] device view of a scalar field (row = env * n_agents + agent)."""
        return self._scal[self.FIELDS.index(name)]

    # ---- reference :175-184
    def store(self, **step_data):
        t, R = self.ptr, self._rows
        scal = np.concatenate([self._per_agent(step_data[k]).reshape(1, R) for k in self.FIELDS[:self.STORED]])
        obs = self._per_agent(step_data['obs'])
        scal_d = torch.from_numpy(np.ascontiguousarray(scal)).to(self.device)
        obs_d = torch.from_numpy(np.ascontiguousarray(obs)).to(self.device)
        _lib.call("xb_rollout_store", _lib.ptr(self._obs), _lib.ptr(obs_d), self._obs_dim * 4, _lib.ptr(self._scal),
                  _lib.ptr(scal_d), self.STORED, R, self.n_size, t)
        if self.use_actions_mask:
            av = np.zeros((R, _pad4(self._n_act)), np.uint8)
            av[:, :self._n_act] = self._per_agent(step_data['avail_actions'], np.float32) != 0
            av_d = torch.from_numpy(av).to(self.device)
            _lib.call("xb_rollout_store", _lib.ptr(self._avail), _lib.ptr(av_d), av.shape[1], None, None, 0, R,
                      self.n_size, t)
        if self.store_global_state:
            st_d = torch.from_numpy(np.ascontiguousarray(step_data['state'], dtype=np.float32)).to(self.device)
            _lib.call("xb_rollout_store", _lib.ptr(self._state), _lib.ptr(st_d), self._state_dim * 4, None, None, 0,
                      self.n_envs, self.n_size, t)
        self.ptr = (self.ptr + 1) % self.n_size
        self.size = min(self.size + 1, self.n_size)

    # ---- reference :186-240
    def finish_path(self, i_env=None, agent_grouping=None, value_next=None, value_normalizer=None, **kwargs):
        if self.size == 0:
            return
        beg = int(self.start_ids[i_env])
        end = self.n_size if self.full else self.ptr
        if end > beg:
            n = self.n_agents
            rows = slice(i_env * n, (i_env + 1) * n)
            self._seg_end[rows, end - 1] = 1
            self._boot[rows, end - 1] = [np.float32(value_next[k]) for k in self.agent_keys]
            self._seg_end_d[rows].copy_(torch.from_numpy(self._seg_end[rows]))
            self._boot_d[rows].copy_(torch.from_numpy(self._boot[rows]))
            self._start_d[rows].fill_(beg)
            self._cov_d[rows].fill_(end)
            self._gae(rows, self._seg_end_d[rows], self._boot_d[rows], self._start_d[rows], self._cov_d[rows],
                      agent_grouping, value_normalizer)
        self.start_ids[i_env] = self.ptr

    # ---- reference :242-270
    def sample(self, indexes=None):
        assert self.full, "Not enough transitions for on-policy buffer to random sample."
        idx = np.asarray(indexes, dtype=np.int64).reshape(-1)
        B, n, T = idx.size, self.n_agents, self.n_size
        env, step = np.divmod(idx, T)
        slots = ((env[None, :] * n + np.arange(n)[:, None]) * T + step[None, :]).reshape(-1)   # agent-major
        slot_t = torch.from_numpy(slots).to(self.device)
        F = len(self.FIELDS)
        scal = torch.empty((F, n * B), dtype=torch.float32, device=self.device)
        stats = torch.empty(2, dtype=torch.float32, device=self.device)
        _lib.call("xb_gather_scalars", _lib.ptr(self._scal), self._rows * T, _lib.ptr(slot_t), n * B, F,
                  _lib.ptr(scal), -1, _lib.ptr(stats), _lib.ptr(self._scratch))
        if self.use_advantage_norm:
            adv_plane, ia = self._scal[F - 1], F - 1
            for k in range(n):
                _lib.call("xb_gather_scalars", _lib.ptr(adv_plane), self._rows * T, _lib.ptr(slot_t[k * B:]), B, 1,
                          _lib.ptr(scal[ia, k * B:]), 0, _lib.ptr(stats), _lib.ptr(self._scratch))
        st = {name: scal[i] for i, name in enumerate(self.FIELDS)}
        st['obs'] = self._gather_rows(self._obs.flatten(0, 1), slot_t)         # one gathered row per (row, step) slot
        if self.use_actions_mask:
            st['avail_actions'] = self._gather_rows(self._avail.flatten(0, 1), slot_t)
        if self.store_global_state:
            s_idx = torch.from_numpy(np.tile(env * T + step, n)).to(self.device)
            st['state'] = self._gather_rows(self._state.flatten(0, 1), s_idx)
        return dict(self._split(st, B), batch_size=B, _stacked=st)

    # ---- checkpoint (the reference does not save its rollout)
    def state_dict(self):
        return {"class": type(self).__name__, "buffer_size": self.buffer_size, "n_envs": self.n_envs,
                "ptr": int(self.ptr), "size": int(self.size), "start_ids": self.start_ids.copy(),
                "scal": self._scal.cpu(), "obs": self._obs.cpu(),
                "avail": None if self._avail is None else self._avail.cpu(),
                "state": None if self._state is None else self._state.cpu(),
                "seg_end": self._seg_end.copy(), "boot": self._boot.copy()}

    def load_state_dict(self, sd):
        if (sd.get("class"), sd.get("buffer_size"), sd.get("n_envs")) != (type(self).__name__, self.buffer_size,
                                                                           self.n_envs):
            raise ValueError("on-policy MARL checkpoint does not match this buffer's size / envs")
        self._scal.copy_(sd["scal"])
        self._obs.copy_(sd["obs"])
        if self._avail is not None:
            self._avail.copy_(sd["avail"])
        if self._state is not None:
            self._state.copy_(sd["state"])
        self._seg_end[:] = sd["seg_end"]
        self._boot[:] = sd["boot"]
        self.ptr, self.size, self.start_ids = int(sd["ptr"]), int(sd["size"]), np.array(sd["start_ids"])


class MARL_OnPolicyBuffer_RNN(_MARLOnPolicyBuffer):
    """Episode-major on-policy rollout for recurrent MAPPO - mirror of MARL_OnPolicyBuffer_RNN
    (xuance/common/memory_tools_marl.py:273-515): same constructor arguments, keys, ``ptr / size / full``, ``clear /
    clear_episodes / store / store_episodes / finish_path / sample``.  ``buffer_size`` counts episodes.

    Everything lives in HBM.  The per-env staging rows are (env, agent) pairs over ``T_max = max_episode_steps``; each
    vector step is one ``xb_rollout_store_at`` launch per array, at each env's own episode step.  ``finish_path`` runs
    ``xb_gae_scan_vn`` over env i's rows on ``[0, min(i_step, T_max))`` with the ValueNorm state of that moment, then
    copies the rows into ring slot ``ptr`` and clears only that env's ``filled``: as in the reference, the staging is
    never zeroed between episodes, so the padded tail of an env's second episode still holds its first episode's data.
    ``sample`` gathers whole episodes with K3 into sequence-major ``[B*n, T, .]`` (sequence k*B + b is agent k of
    episode b) and does not normalise advantages (the reference's recurrent ``sample`` does not either)."""
    BOX_REFUSAL = "MARL_OnPolicyBuffer_RNN: Box action spaces (Gaussian MAPPO) are not supported"

    def __init__(self, agent_keys, state_space=None, obs_space=None, act_space=None, n_envs=1, buffer_size=1,
                 max_episode_steps=1, use_gae=False, use_advnorm=False, gamma=None, gae_lam=None, device="cuda:0",
                 **kwargs):
        super().__init__(agent_keys, state_space, obs_space, act_space, n_envs, buffer_size, use_gae, use_advnorm,
                         gamma, gae_lam, device, **kwargs)
        self.max_eps_len = max_episode_steps
        self._a4 = _pad4(self._n_act)
        self._seg_end = np.zeros((self._rows, self.max_eps_len), np.uint8)
        self._boot = np.zeros((self._rows, self.max_eps_len), np.float32)
        self.clear()
        self.clear_episodes()

    @property
    def data_keys(self):
        keys = ['obs'] + list(self.FIELDS) + ['filled']
        if self.store_global_state:
            keys.append('state')
        if self.use_actions_mask:
            keys.append('avail_actions')
        return keys

    @property
    def full(self):
        return self.size >= self.buffer_size

    def clear(self):
        """The episode ring: scalars [buffer_size * n, F, T] (row = slot * n + agent), obs [buffer_size * n, T, obs],
        filled [buffer_size, T]."""
        S, T, dev = self.buffer_size * self.n_agents, self.max_eps_len, self.device
        self._scal = torch.zeros((S, len(self.FIELDS), T), dtype=torch.float32, device=dev)
        self._obs = torch.zeros((S, T, self._obs_dim), dtype=torch.float32, device=dev)
        self._avail = torch.zeros((S, T, self._a4), dtype=torch.uint8, device=dev) if self.use_actions_mask else None
        self._state = (torch.zeros((self.buffer_size, T, self._state_dim), dtype=torch.float32, device=dev)
                       if self.store_global_state else None)
        self._filled = torch.zeros((self.buffer_size, T), dtype=torch.float32, device=dev)
        self.ptr, self.size = 0, 0

    def clear_episodes(self):
        """The per-env staging: scalars [F, n_envs * n, T] (K1's layout), obs [n_envs * n, T, obs], filled [n_envs, T]."""
        R, T, dev = self._rows, self.max_eps_len, self.device
        self._ep_scal = torch.zeros((len(self.FIELDS), R, T), dtype=torch.float32, device=dev)
        self._ep_obs = torch.zeros((R, T, self._obs_dim), dtype=torch.float32, device=dev)
        self._ep_avail = torch.zeros((R, T, self._a4), dtype=torch.uint8, device=dev) if self.use_actions_mask else None
        self._ep_state = (torch.zeros((self.n_envs, T, self._state_dim), dtype=torch.float32, device=dev)
                          if self.store_global_state else None)
        self._ep_filled = torch.zeros((1, self.n_envs, T), dtype=torch.float32, device=dev)
        self._ones = torch.ones((1, self.n_envs), dtype=torch.float32, device=dev)

    def field(self, name):
        """[n_envs * n_agents, T] device view of a staging scalar field (row = env * n_agents + agent)."""
        return self._ep_scal[self.FIELDS.index(name)]

    # ---- reference :397-414
    def store(self, **step_data):
        T, R = self.max_eps_len, self._rows
        steps = np.asarray(step_data['episode_steps'], np.int32).reshape(self.n_envs)
        steps_env = torch.from_numpy(steps).to(self.device)
        steps_row = torch.from_numpy(np.repeat(steps, self.n_agents)).to(self.device)
        scal = np.concatenate([self._per_agent(step_data[k]).reshape(1, R) for k in self.FIELDS[:self.STORED]])
        scal_d = torch.from_numpy(np.ascontiguousarray(scal)).to(self.device)
        obs_d = torch.from_numpy(np.ascontiguousarray(self._per_agent(step_data['obs']))).to(self.device)
        _lib.call("xb_rollout_store_at", _lib.ptr(self._ep_obs), _lib.ptr(obs_d), self._obs_dim * 4,
                  _lib.ptr(self._ep_scal), _lib.ptr(scal_d), self.STORED, R, T, _lib.ptr(steps_row))
        if self.use_actions_mask:
            av = np.zeros((R, self._a4), np.uint8)
            av[:, :self._n_act] = self._per_agent(step_data['avail_actions'], np.float32) != 0
            av_d = torch.from_numpy(av).to(self.device)
            _lib.call("xb_rollout_store_at", _lib.ptr(self._ep_avail), _lib.ptr(av_d), self._a4, None, None, 0, R, T,
                      _lib.ptr(steps_row))
        st_d = None
        if self.store_global_state:
            st_d = torch.from_numpy(np.ascontiguousarray(step_data['state'], dtype=np.float32)).to(self.device)
        # filled[env, step] = 1, in the same launch as the global state rows
        _lib.call("xb_rollout_store_at", _lib.ptr(self._ep_state), _lib.ptr(st_d), self._state_dim * 4,
                  _lib.ptr(self._ep_filled), _lib.ptr(self._ones), 1, self.n_envs, T, _lib.ptr(steps_env))

    # ---- reference :416-435: env i's staging rows -> ring slot ptr (device copies), then clear only its `filled`
    def store_episodes(self, i_env):
        n, p = self.n_agents, self.ptr
        rows = slice(i_env * n, (i_env + 1) * n)
        self._scal[p * n:(p + 1) * n].copy_(self._ep_scal[:, rows].transpose(0, 1))
        self._obs[p * n:(p + 1) * n].copy_(self._ep_obs[rows])
        if self.use_actions_mask:
            self._avail[p * n:(p + 1) * n].copy_(self._ep_avail[rows])
        if self.store_global_state:
            self._state[p].copy_(self._ep_state[i_env])
        self._filled[p].copy_(self._ep_filled[0, i_env])
        self.ptr = (self.ptr + 1) % self.buffer_size
        self.size = min(self.size + 1, self.buffer_size)
        self._ep_filled[0, i_env].zero_()

    # ---- reference :437-490
    def finish_path(self, i_env=None, i_step=None, agent_grouping=None, value_next=None, value_normalizer=None,
                    **kwargs):
        n = self.n_agents
        env_step = min(int(i_step), self.max_eps_len)
        if env_step > 0:
            rows = slice(i_env * n, (i_env + 1) * n)
            self._seg_end[rows] = 0
            self._seg_end[rows, env_step - 1] = 1
            self._boot[rows] = 0
            self._boot[rows, env_step - 1] = [np.float32(value_next[k]) for k in self.agent_keys]
            seg_d = torch.from_numpy(self._seg_end[rows]).to(self.device)
            boot_d = torch.from_numpy(self._boot[rows]).to(self.device)
            cov_d = torch.full((n,), env_step, dtype=torch.int32, device=self.device)
            self._gae(rows, seg_d, boot_d, None, cov_d, agent_grouping, value_normalizer)
        self.store_episodes(i_env)

    # ---- reference :492-515
    def sample(self, indexes=None):
        assert self.full, "Not enough transitions for on-policy buffer to random sample"
        idx = np.asarray(indexes, dtype=np.int64).reshape(-1)
        B, n, T = idx.size, self.n_agents, self.max_eps_len
        seq = (idx[None, :] * n + np.arange(n)[:, None]).reshape(-1)                # agent-major: k * B + b
        seq_t = torch.from_numpy(seq).to(self.device)
        ep_t = torch.from_numpy(np.tile(idx, n)).to(self.device)
        scal = self._gather_rows(self._scal, seq_t)
        st = {name: scal[:, i].contiguous() for i, name in enumerate(self.FIELDS)}    # [n*B, T]
        st['obs'] = self._gather_rows(self._obs, seq_t)
        st['filled'] = self._gather_rows(self._filled, ep_t)
        if self.use_actions_mask:
            st['avail_actions'] = self._gather_rows(self._avail, seq_t)
        if self.store_global_state:
            st['state'] = self._gather_rows(self._state, ep_t)
        return dict(self._split(st, B), batch_size=B, sequence_length=T, _stacked=st)

    # ---- checkpoint (the reference does not save its rollout)
    def state_dict(self):
        t = lambda x: None if x is None else x.cpu()
        return {"class": type(self).__name__, "buffer_size": self.buffer_size, "n_envs": self.n_envs,
                "max_eps_len": self.max_eps_len, "ptr": int(self.ptr), "size": int(self.size),
                "data": {k: t(getattr(self, k)) for k in ("_scal", "_obs", "_avail", "_state", "_filled")},
                "episode_data": {k: t(getattr(self, k)) for k in ("_ep_scal", "_ep_obs", "_ep_avail", "_ep_state",
                                                                  "_ep_filled")}}

    def load_state_dict(self, sd):
        if (sd.get("class"), sd.get("buffer_size"), sd.get("n_envs"), sd.get("max_eps_len")) != \
                (type(self).__name__, self.buffer_size, self.n_envs, self.max_eps_len):
            raise ValueError("recurrent on-policy MARL checkpoint does not match this buffer's size / envs / length")
        for group in ("data", "episode_data"):
            for k, v in sd[group].items():
                dst = getattr(self, k)
                if dst is not None:
                    dst.copy_(v)
        self.ptr, self.size = int(sd["ptr"]), int(sd["size"])

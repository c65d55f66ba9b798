"""Multi-agent on-policy agents - mirrors of

* ``OnPolicyMARLAgents``  xuance/torch/agents/core/on_policy_marl.py:16-693 (``store_experience``, ``get_actions``
                          returning values and log-probabilities, ``values_next``, ``train``, ``run_episodes``,
                          ``train_epochs``, ``test``), the feed-forward branch (``use_rnn=False``);
* ``MAPPO_Agents``        xuance/torch/agents/multi_agent_rl/mappo_agents.py:18-112.

Scope: one parameter-sharing group, Discrete actions (with or without action masks), Basic_MLP representations or,
with ``use_rnn=True``, the LayerNorm Basic_RNN whose GRU runs on K13 (``Basic_RNN_K13``).  The recurrent branch is the
reference's: ``train`` repeats ``run_episodes(n_envs)`` -> ``train_epochs``; the actor and critic hidden states live on
the device as [1, n_envs * n_agents, H] and a finished env's rows are zeroed there; acting runs K13 with T = 1 from the
carried states.
Acting: one staged upload of the vector step's observations ([n_envs * n_agents, obs_dim]), the actor, the mask as
-1e10 logits (actor_head.py:40), K10 sampling on the device, the critic, and ONE device-to-host read of actions,
log-probabilities and values."""
from copy import deepcopy
from operator import itemgetter

import numpy as np
import torch
import torch.nn as nn

from ... import _lib
from ...common import MARL_OnPolicyBuffer, MARL_OnPolicyBuffer_RNN
from ..rl_models import CategoricalActor, CentralizedStateValueCritic, MultiAgentActorCritic
from .marl import MARLAgents, MARLActionOutput


class OnPolicyMARLAgents(MARLAgents):
    """on_policy_marl.py:16-693."""

    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        super().__init__(config, envs, num_agents, agent_keys, state_space, observation_space, action_space, callback)
        self.on_policy = True
        self.continuous_control = False
        self.n_epochs, self.n_minibatch = config.n_epochs, config.n_minibatch
        self.buffer_size = config.buffer_size
        self.batch_size = self.buffer_size // self.n_minibatch

    def _build_memory(self):
        """on_policy_marl.py:77-98."""
        avail_shape = {k: (self.action_space[k].n,) for k in self.agent_keys} if self.use_actions_mask else None
        if self.use_rnn:
            return MARL_OnPolicyBuffer_RNN(agent_keys=self.agent_keys,
                                           state_space=self.state_space if self.use_global_state else None,
                                           obs_space=self.observation_space, act_space=self.action_space,
                                           n_envs=self.n_envs, buffer_size=self.config.buffer_size,
                                           max_episode_steps=self.episode_length, use_gae=self.config.use_gae,
                                           use_advnorm=self.config.use_advnorm, gamma=self.config.gamma,
                                           gae_lam=self.config.gae_lambda, avail_actions_shape=avail_shape,
                                           use_actions_mask=self.use_actions_mask, device=self.device)
        return MARL_OnPolicyBuffer(agent_keys=self.agent_keys,
                                   state_space=self.state_space if self.use_global_state else None,
                                   obs_space=self.observation_space, act_space=self.action_space, n_envs=self.n_envs,
                                   buffer_size=self.config.buffer_size, use_gae=self.config.use_gae,
                                   use_advnorm=self.config.use_advnorm, gamma=self.config.gamma,
                                   gae_lam=self.config.gae_lambda, avail_actions_shape=avail_shape,
                                   use_actions_mask=self.use_actions_mask, max_episode_steps=self.episode_length,
                                   device=self.device)

    def store_experience(self, obs_list, avail_actions, actions_list, log_pi_a, rewards_list, values_dict,
                         terminals_list, info, **kwargs):
        """on_policy_marl.py:103-158."""
        data = {'obs': self._agent_arrays(obs_list), 'actions': self._agent_arrays(actions_list),
                'log_pi_old': log_pi_a, 'rewards': self._agent_arrays(rewards_list), 'values': values_dict,
                'terminals': self._agent_arrays(terminals_list),
                'agent_mask': self._agent_arrays([d['agent_mask'] for d in info])}
        if self.use_global_state:
            data['state'] = np.array(kwargs['state'])
        if self.use_actions_mask:
            data['avail_actions'] = self._agent_arrays(avail_actions)
        if self.use_rnn:
            data['episode_steps'] = np.array([d['episode_step'] - 1 for d in info])
        self.memory.store(**data)

    def _states(self, state, n_envs):
        if not self.use_global_state or state is None:
            return None
        s = torch.as_tensor(np.asarray(state, np.float32), device=self.device)
        return s.repeat_interleave(self.n_agents, dim=0)          # rows are env-major, agent-minor

    def _critic_values(self, obs_d, state, n_envs, rnn_states=None, return_states=False):
        """The values of the acting rows [n_envs * n_agents] (and the new critic states with return_states)."""
        return self.model.values(obs_d, self._states(state, n_envs), rnn_states=rnn_states, return_states=return_states)

    def _build_agent_feature_encoder(self, representation_choice, group_agents, input_space):
        if not self.use_rnn:
            return super()._build_agent_feature_encoder(representation_choice, group_agents, input_space)
        if representation_choice != "Basic_RNN":
            raise NotImplementedError("use_rnn=True takes representation: Basic_RNN, got %s" % representation_choice)
        return self._build_k13_encoder(input_space, self.normalize_fn)

    @torch.no_grad()
    def get_actions(self, obs_list, state=None, avail_actions_list=None, rnn_states_actor=None,
                    rnn_states_critic=None, test_mode=False, deterministic=False, **kwargs):
        """on_policy_marl.py:207-306."""
        n_envs, K = len(obs_list), self.agent_keys
        obs, avail = self._build_inputs(obs_list, avail_actions_list)
        obs_d = torch.from_numpy(obs).to(self.device)
        if self.use_rnn:
            logits, rnn_states_actor = self.model.logits(obs_d, rnn_states=rnn_states_actor, return_states=True)
        else:
            logits = self.model.logits(obs_d)
        out, rnn_states_critic = self._act(obs_d, logits, avail, state, n_envs, rnn_states_critic, test_mode,
                                           deterministic)
        host = out.cpu().numpy().reshape(3, n_envs, len(K))
        actions_list = [{k: int(host[0, e, i]) for i, k in enumerate(K)} for e in range(n_envs)]
        log_pi, values = {}, {}
        if not test_mode:
            log_pi = {k: host[1, :, i].copy() for i, k in enumerate(K)}
            values = {k: host[2, :, i].copy() for i, k in enumerate(K)}
        return MARLActionOutput(env_actions=actions_list, log_probs=log_pi, values=values,
                                rnn_states_actor=rnn_states_actor, rnn_states_critic=rnn_states_critic)

    def _act(self, obs_d, logits, avail, state, n_envs, rnn_states_critic, test_mode, deterministic):
        """K10 samples the rows' actions from the actor's logits -> ([3, R] actions, log-probabilities and, outside
        test_mode, the critic's values; the new critic states)."""
        if avail is not None:
            logits = logits.masked_fill(torch.from_numpy(avail).to(self.device) == 0, -1e10)
        logits = logits.contiguous()
        R, A = logits.shape
        out = torch.empty((3, R), dtype=torch.float32, device=self.device)   # actions, log_pi, values
        acts_i = torch.empty(R, dtype=torch.int32, device=self.device)
        u = None if deterministic else torch.rand(R, device=self.device)
        _lib.call("xb_categorical_act", _lib.ptr(logits), _lib.ptr(u), None, R, A, _lib.ptr(out[0]), _lib.ptr(acts_i),
                  _lib.ptr(out[1]), None)
        if not test_mode:
            if self.use_rnn:
                out[2], rnn_states_critic = self._critic_values(obs_d, state, n_envs, rnn_states_critic, True)
            else:
                out[2] = self._critic_values(obs_d, state, n_envs)
        return out, rnn_states_critic

    @torch.no_grad()
    def values_next(self, i_env, obs_dict, state=None, rnn_states_critic=None):
        """on_policy_marl.py:308-357."""
        obs, _ = self._build_inputs([obs_dict])
        st = None if state is None else np.asarray(state)[None]
        h = None
        if self.use_rnn:      # the critic rows of env i (on_policy_marl.py:337-344)
            n = len(self.agent_keys)
            h = rnn_states_critic[:, i_env * n:(i_env + 1) * n]
        v = self._critic_values(torch.from_numpy(obs).to(self.device), st, 1, h).cpu().numpy()
        return None, {k: v[i] for i, k in enumerate(self.agent_keys)}

    def init_rnn_states(self, n_envs):
        """on_policy_marl.py:160-178: zero actor / critic states for n_envs envs (None without recurrence)."""
        if not self.use_rnn:
            return None, None
        return self.model.init_rnn_states(n_envs * len(self.agent_keys))

    def init_rnn_states_item(self, i_env, rnn_states_actor=None, rnn_states_critic=None):
        """on_policy_marl.py:180-205: zero env i_env's rows."""
        if not self.use_rnn:
            return rnn_states_actor, rnn_states_critic
        n = len(self.agent_keys)
        return self.model.init_rnn_states_item(slice(i_env * n, (i_env + 1) * n), rnn_states_actor, rnn_states_critic)

    def _finish(self, i, terminated, next_obs, next_state):
        if all(terminated.values()):
            value_next = {k: 0.0 for k in self.agent_keys}
        else:
            _, value_next = self.values_next(i_env=i, obs_dict=next_obs, state=next_state)
        self.memory.finish_path(i_env=i, agent_grouping=self.agent_grouping, value_next=value_next,
                                value_normalizer=self.learner.value_normalizer)

    def train(self, train_steps):
        """on_policy_marl.py:384-482."""
        train_info = {}
        if self.use_rnn:        # :384-403: whole episodes, then the epochs
            step_start = self.current_step
            while self.current_step - step_start < train_steps * self.n_envs:
                self.run_episodes(n_episodes=self.n_envs, test_mode=False, close_envs=False)
                update_info = self.train_epochs(n_epochs=self.n_epochs)
                self.log_infos(update_info, self.current_step)
                train_info.update(update_info)
            self.callback.on_train_step_end(self.current_step, envs=self.train_envs, policy=self.model,
                                            train_steps=train_steps, train_info=train_info)
            return train_info
        envs = self.train_envs
        obs_list = envs.buf_obs
        avail_actions = envs.buf_avail_actions if self.use_actions_mask else None
        state = envs.buf_state if self.use_global_state else None
        for _ in range(train_steps):
            policy_out = self.get_actions(obs_list=obs_list, state=state, avail_actions_list=avail_actions)
            actions_list = policy_out.env_actions
            next_obs_list, rewards_list, terminated_list, truncated, info = envs.step(actions_list)
            next_state = envs.buf_state if self.use_global_state else None
            next_avail_actions = envs.buf_avail_actions if self.use_actions_mask else None
            self.callback.on_train_step(self.current_step, envs=envs, policy=self.model, obs=obs_list,
                                        policy_out=policy_out, acts=actions_list, next_obs=next_obs_list,
                                        rewards=rewards_list, state=state, next_state=next_state,
                                        avail_actions=avail_actions, next_avail_actions=next_avail_actions,
                                        terminals=terminated_list, truncations=truncated, infos=info,
                                        train_steps=train_steps, values_dict=policy_out.values)
            self.store_experience(obs_list, avail_actions, actions_list, policy_out.log_probs, rewards_list,
                                  policy_out.values, terminated_list, info, state=state)
            if self.memory.full:
                for i in range(self.n_envs):
                    self._finish(i, terminated_list[i], next_obs_list[i],
                                 next_state[i] if self.use_global_state else None)
            update_info = self.train_epochs(n_epochs=self.n_epochs)
            self.log_infos(update_info, self.current_step)
            train_info.update(update_info)
            obs_list, avail_actions = deepcopy(next_obs_list), deepcopy(next_avail_actions)
            state = deepcopy(next_state) if self.use_global_state else None
            for i in range(self.n_envs):
                if all(terminated_list[i].values()) or truncated[i]:
                    self._finish(i, terminated_list[i], obs_list[i], state[i] if self.use_global_state else None)
                    self._reset_env(envs, i, info, obs_list, state, avail_actions)
                    self.current_episode[i] += 1
                    episode_info = {
                        "Train-Results/Episode-Steps": {"env-%d" % i: info[i]["episode_step"]},
                        "Train-Results/Episode-Rewards": {
                            "env-%d" % i: float(np.mean(itemgetter(*self.agent_keys)(info[i]["episode_score"])))}}
                    self.log_infos(episode_info, self.current_step)
                    train_info.update(episode_info)
                    self.callback.on_train_episode_info(envs=envs, policy=self.model, env_id=i, infos=info,
                                                        rank=self.rank, use_wandb=self.use_wandb,
                                                        current_step=self.current_step,
                                                        current_episode=self.current_episode,
                                                        train_steps=train_steps)
            self.current_step += self.n_envs
            self.callback.on_train_step_end(self.current_step, envs=envs, policy=self.model,
                                            train_steps=train_steps, train_info=train_info)
        return train_info

    def run_episodes(self, n_episodes=1, deterministic_policy=False, run_envs=None, test_mode=False, close_envs=True):
        """on_policy_marl.py:484-630 (no rendering)."""
        envs = self.train_envs if run_envs is None else run_envs
        num_envs = envs.num_envs
        _current_episode, scores = 0, []
        obs_list, info = envs.reset()
        avail_actions = envs.buf_avail_actions if self.use_actions_mask else None
        state = envs.buf_state if self.use_global_state else None
        if self.use_rnn and not test_mode:
            self.memory.clear_episodes()        # :523-525: a fresh staging per call (not per episode)
        rnn_states_actor, rnn_states_critic = self.init_rnn_states(num_envs)
        while _current_episode < n_episodes:
            policy_out = self.get_actions(obs_list=obs_list, state=state, avail_actions_list=avail_actions,
                                          rnn_states_actor=rnn_states_actor, rnn_states_critic=rnn_states_critic,
                                          test_mode=test_mode, deterministic=deterministic_policy)
            rnn_states_actor, rnn_states_critic = policy_out.rnn_states_actor, policy_out.rnn_states_critic
            actions_list = policy_out.env_actions
            next_obs_list, rewards_list, terminated_list, truncated, info = envs.step(actions_list)
            next_state = envs.buf_state if self.use_global_state else None
            next_avail_actions = envs.buf_avail_actions if self.use_actions_mask else None
            if not test_mode:
                self.store_experience(obs_list, avail_actions, actions_list, policy_out.log_probs, rewards_list,
                                      policy_out.values, terminated_list, info, state=state)
            obs_list, avail_actions = deepcopy(next_obs_list), deepcopy(next_avail_actions)
            state = deepcopy(next_state) if self.use_global_state else None
            for i in range(num_envs):
                if all(terminated_list[i].values()) or truncated[i]:
                    _current_episode += 1
                    scores.append(float(np.mean(itemgetter(*self.agent_keys)(info[i]["episode_score"]))))
                    if not test_mode and self.use_rnn:
                        if all(terminated_list[i].values()):
                            value_next = {k: 0.0 for k in self.agent_keys}
                        else:
                            _, value_next = self.values_next(i_env=i, obs_dict=obs_list[i],
                                                             state=None if state is None else state[i],
                                                             rnn_states_critic=rnn_states_critic)
                        self.memory.finish_path(i_env=i, i_step=info[i]['episode_step'],
                                                agent_grouping=self.agent_grouping, value_next=value_next,
                                                value_normalizer=self.learner.value_normalizer)
                    if self.use_rnn:
                        rnn_states_actor, rnn_states_critic = self.init_rnn_states_item(
                            i, rnn_states_actor, None if test_mode else rnn_states_critic)
                    if not test_mode:
                        if not self.use_rnn:
                            self._finish(i, terminated_list[i], obs_list[i], None if state is None else state[i])
                        self.current_step += info[i]["episode_step"]
                        self.callback.on_train_episode_info(envs=envs, policy=self.model, env_id=i, infos=info,
                                                            rank=self.rank, use_wandb=self.use_wandb,
                                                            current_step=self.current_step,
                                                            current_episode=self.current_episode,
                                                            n_episodes=n_episodes)
                    self._reset_env(envs, i, info, obs_list, state, avail_actions)
        if test_mode:
            self.log_infos({"Test-Results/Episode-Rewards/Mean-Score": float(np.mean(scores)),
                            "Test-Results/Episode-Rewards/Std-Score": float(np.std(scores))}, self.current_step)
            if close_envs:
                envs.close()
        return scores

    def train_epochs(self, n_epochs=1):
        """on_policy_marl.py:632-661: shuffled n_minibatch slices per epoch; the info of the last update (only that
        one reads the device statistics back)."""
        info_train = {}
        if self.memory.full:       # buffer_size counts steps per env-row, or episodes with use_rnn
            indexes = np.arange(self.buffer_size)
            for e in range(n_epochs):
                np.random.shuffle(indexes)
                for start in range(0, self.buffer_size, self.batch_size):
                    last = e == n_epochs - 1 and start + self.batch_size >= self.buffer_size
                    info_train = self._update(self.memory.sample(indexes[start:start + self.batch_size]), last)
            self.callback.on_train_epochs_end(self.current_step, policy=self.model, memory=self.memory,
                                              current_episode=self.current_episode, n_epochs=n_epochs,
                                              buffer_size=self.buffer_size, update_info=info_train)
            self.memory.clear()
        return info_train

    def _update(self, sample, sync):
        return self.learner.update(sample, sync=sync)

    def test(self, test_episodes, deterministic_policy=True, test_envs=None, close_envs=True):
        return self.run_episodes(n_episodes=test_episodes, run_envs=test_envs, test_mode=True,
                                 deterministic_policy=deterministic_policy, close_envs=close_envs)


class MAPPO_Agents(OnPolicyMARLAgents):
    """mappo_agents.py:18-112."""

    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        super().__init__(config, envs, num_agents, agent_keys, state_space, observation_space, action_space, callback)
        if not all(hasattr(self.action_space[k], "n") for k in self.agent_keys):
            raise NotImplementedError("Gaussian MAPPO (Box action spaces) is not supported: MAPPO here takes Discrete "
                                      "action spaces")
        self.model = self._build_model()
        self.memory = self._build_memory()
        self.learner = self._build_learner(self.config, self.agent_grouping, self.model, self.callback)

    def _build_model(self):
        actors, critics, critic_encoders = nn.ModuleDict(), nn.ModuleDict(), nn.ModuleDict()
        for group_key, group_agents in self.groups.items():
            ref = group_agents[0]
            enc = self._build_agent_feature_encoder(self.config.representation, group_agents,
                                                    self.observation_space[ref])
            actors[group_key] = CategoricalActor(representation=enc, actor_hidden_size=self.config.actor_hidden_size,
                                                 action_space=self.action_space[ref], normalizer=self.normalize_fn,
                                                 initializer=self.initializer, activation=self.activation,
                                                 device=self.device)
            critic_encoders[group_key] = self._build_agent_feature_encoder(self.config.representation, group_agents,
                                                                           self.observation_space[ref])
        for group_key in self.groups:
            critics[group_key] = CentralizedStateValueCritic(
                grouping=self.agent_grouping, representations=critic_encoders,
                state_space=self.state_space if self.use_global_state else None,
                critic_hidden_size=self.config.critic_hidden_size, normalizer=self.normalize_fn,
                initializer=self.initializer, activation=self.activation, device=self.device)
        return MultiAgentActorCritic(grouping=self.agent_grouping, actors=actors, critics=critics,
                                     use_rnn=self.use_rnn, device=self.device).to(self.device)


class IPPO_Agents(OnPolicyMARLAgents):
    def __init__(self, config, *args, **kwargs):
        raise NotImplementedError("IPPO is not supported yet (MAPPO's loss kernel with a per-agent critic input; "
                                  "DESIGN.md section 9)")

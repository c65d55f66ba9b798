"""Multi-agent agents of the QMIX path - mirrors of

* ``MARLAgents``           xuance/torch/agents/base/agents_marl.py:26-330 (construction from vector envs or explicit
                           spaces, agent grouping, model / learner builders, save / load, logging);
* ``OffPolicyMARLAgents``  xuance/torch/agents/core/off_policy_marl.py:17-622 (``store_experience``, RNN state
                           helpers, epsilon-greedy ``exploration``, ``get_actions``, ``train``, ``run_episodes``,
                           ``train_epochs``, ``test``);
* ``QMIX_Agents``          xuance/torch/agents/multi_agent_rl/qmix_agents.py:12-93.

Scope (DESIGN.md section 8): one parameter-sharing group of GRU agents with discrete actions (``use_rnn=True``,
``use_parameter_sharing=True``) - the configuration of BASELINE config 5.  The environment interface is the
reference's: per-env lists of per-agent dicts.  What differs underneath: a vector step's observations go to the device
in ONE staged upload ([n_envs * n_agents, obs_dim]), the GRU step + masked arg-max run there and ONE small D2H returns
the greedy actions; finished episodes are ingested into the HBM episode ring by K1 (common/memory_tools_marl.py)."""
import os
from copy import deepcopy
from operator import itemgetter

import numpy as np
import torch
import torch.nn as nn

from ...common import AgentGrouping, BaseCallback, MARL_OffPolicyBuffer_RNN, space2shape
from ..rl_models import (REGISTRY_Representation, ActivationFunctions, AgentFeatureEncoder, Basic_RNN_K13,
                         DiscreteActionValueCritic, QMIX_Mixer, VDN_mixer, MixingQNetwork)
from .agent import set_seed, set_device, InitializeFunctions, NormalizeFunctions
from ..utils import init_distributed_mode


class MARLActionOutput:
    """What ``get_actions`` returns: the off-policy agents fill ``rnn_states``, the on-policy ones ``log_probs``,
    ``values`` and the actor / critic states."""

    def __init__(self, env_actions=None, rnn_states=None, values=None, log_probs=None, rnn_states_actor=None,
                 rnn_states_critic=None):
        self.env_actions, self.rnn_states, self.values, self.log_probs = env_actions, rnn_states, values, log_probs
        self.rnn_states_actor, self.rnn_states_critic = rnn_states_actor, rnn_states_critic


class MARLAgents:
    """agents_marl.py:26-330."""

    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        set_seed(config.seed)
        self.config = config
        self.use_rnn = getattr(config, "use_rnn", False)
        self.use_parameter_sharing = getattr(config, "use_parameter_sharing", True)
        self.use_actions_mask = getattr(config, "use_actions_mask", False)
        self.use_global_state = getattr(config, "use_global_state", False)
        self.distributed_training = getattr(config, "distributed_training", False)
        if self.distributed_training:
            self.rank, self.world_size, local_rank = init_distributed_mode(getattr(config, "master_port", None))
            if torch.cuda.is_available():
                config.device = "cuda:%d" % local_rank
        else:
            self.world_size, self.rank = 1, 0
        self.gamma = config.gamma
        self.start_training = getattr(config, "start_training", 1)
        self.training_frequency = getattr(config, "training_frequency", 1)
        self.n_epochs = getattr(config, "n_epochs", 1)
        self.device = self.config.device = set_device(config.device)
        if torch.device(self.device).type == "cuda":
            torch.cuda.set_device(torch.device(self.device))
        self.train_envs = envs
        self.render = getattr(config, "render", False)
        self.fps = getattr(config, "fps", 15)
        if envs is None:
            if observation_space is None or action_space is None or agent_keys is None or num_agents is None:
                raise ValueError("Please provide the num_agents, agent_keys, observation_space, and action_space when "
                                 "the envs is not provided. Or the networks cannot be built.")
            assert config.parallels % self.world_size == 0
            self.n_envs = config.parallels // self.world_size
            self.n_agents = config.n_agents = num_agents
            self.agent_keys = list(agent_keys)
            self.state_space = state_space
            self.observation_space, self.action_space = observation_space, action_space
            self.episode_length = getattr(config, "episode_length", None)
        else:
            try:
                envs.reset()
            except Exception:
                pass
            self.n_agents = config.n_agents = envs.num_agents
            self.n_envs = envs.num_envs
            self.agent_keys = list(envs.agents)
            self.state_space = envs.state_space
            self.observation_space, self.action_space = envs.observation_space, envs.action_space
            self.episode_length = getattr(config, "episode_length", None) or envs.max_episode_steps
        config.episode_length = self.episode_length
        self.current_step = 0
        self.current_episode = np.zeros((self.n_envs,), np.int32)
        if not self.use_parameter_sharing:
            raise NotImplementedError("hot-path scope: one parameter-sharing group (use_parameter_sharing=True)")
        self.agent_grouping = AgentGrouping.shared(self.agent_keys)
        self.groups, self.group_keys = self.agent_grouping.groups, self.agent_grouping.group_keys
        self.n_group_agents = {k: len(self.groups[k]) for k in self.group_keys}
        self.normalize_fn = NormalizeFunctions[config.normalize] if hasattr(config, "normalize") else None
        self.initializer = InitializeFunctions[getattr(config, "initializer", "orthogonal")]
        self.activation = ActivationFunctions[config.activation]
        self.model_dir_load = getattr(config, "model_dir", "models")
        self.model_dir_save = os.path.join(os.getcwd(), getattr(config, "model_dir", "models"), f"seed_{config.seed}")
        self.logged, self.writer, self.use_wandb = {}, None, False
        if getattr(config, "logger", None) == "tensorboard" and self.rank == 0:
            try:
                from torch.utils.tensorboard import SummaryWriter
                log_dir = os.path.join(os.getcwd(), getattr(config, "log_dir", "logs"), f"seed_{config.seed}")
                os.makedirs(log_dir, exist_ok=True)
                self.writer = SummaryWriter(log_dir)
            except Exception:
                self.writer = None
        self.model_keys = [self.agent_keys[0]]
        self.model = self.learner = self.memory = None
        self.callback = callback or BaseCallback()

    def log_infos(self, info, x_index):
        for k, v in info.items():
            if v is None:
                continue
            self.logged[k] = v
            if self.writer is not None:
                try:
                    self.writer.add_scalars(k, v, x_index) if isinstance(v, dict) else self.writer.add_scalar(k, v, x_index)
                except Exception:
                    pass

    def log_videos(self, info, fps, x_index=0):
        pass

    def save_model(self, model_name, model_path=None):
        if self.distributed_training and self.rank > 0:
            return
        model_path = self.model_dir_save if model_path is None else model_path
        os.makedirs(model_path, exist_ok=True)
        self.learner.save_model(os.path.join(model_path, model_name))

    def load_model(self, path, model=None):
        return self.learner.load_model(path, model)

    def _build_representation(self, representation_choice, input_space, config):
        if representation_choice not in REGISTRY_Representation:
            raise AttributeError(f"{representation_choice} is not registered in REGISTRY_Representation.")
        return REGISTRY_Representation[representation_choice](
            input_shape=space2shape(input_space), hidden_sizes=getattr(config, "representation_hidden_size", None),
            normalize=self.normalize_fn, initialize=nn.init.orthogonal_, activation=ActivationFunctions[config.activation],
            fc_hidden_sizes=getattr(config, "fc_hidden_sizes", None),
            N_recurrent_layers=getattr(config, "N_recurrent_layers", 1),
            recurrent_hidden_size=getattr(config, "recurrent_hidden_size", None), rnn=getattr(config, "rnn", "GRU"),
            dropout=getattr(config, "dropout", 0), device=self.device)

    def _build_agent_feature_encoder(self, representation_choice, group_agents, input_space):
        if getattr(self.config, "identity_embedding_mode", "none") != "none":
            raise NotImplementedError("agent-identity embeddings are outside the hot-path scope (mode 'none')")
        return AgentFeatureEncoder(self._build_representation(representation_choice, input_space, self.config))

    def _build_k13_encoder(self, input_space, normalize):
        """The LayerNorm Basic_RNN whose GRU runs on K13; ``normalize`` None builds it without the LayerNorms."""
        return AgentFeatureEncoder(Basic_RNN_K13(
            input_shape=space2shape(input_space), normalize=normalize, initialize=nn.init.orthogonal_,
            activation=self.activation, device=self.device, fc_hidden_sizes=self.config.fc_hidden_sizes,
            recurrent_hidden_size=self.config.recurrent_hidden_size,
            N_recurrent_layers=getattr(self.config, "N_recurrent_layers", 1), rnn=getattr(self.config, "rnn", "GRU"),
            dropout=getattr(self.config, "dropout", 0)))

    def _agent_arrays(self, per_env):
        """Per-env dicts [{agent: x}] -> {agent: array over the envs}."""
        return {k: np.array([d[k] for d in per_env]) for k in self.agent_keys}

    def _reset_env(self, envs, i, info, obs_list, state, avail_actions):
        """A finished env i goes on from what its reset returned (``info[i]["reset_*"]``), in the rollout's lists and
        in the env's buffers."""
        obs_list[i] = envs.buf_obs[i] = info[i]["reset_obs"]
        if self.use_global_state:
            state[i] = envs.buf_state[i] = info[i]["reset_state"]
        if self.use_actions_mask:
            avail_actions[i] = envs.buf_avail_actions[i] = info[i]["reset_avail_actions"]

    def _build_inputs(self, obs_list, avail_actions_list=None):
        """[n_envs * n_agents, obs_dim] (env-major, agent-minor) float32 and the matching uint8 availability rows."""
        K = self.agent_keys
        obs = np.stack([np.stack([np.asarray(d[k], np.float32) for k in K]) for d in obs_list])
        obs = obs.reshape(len(obs_list) * len(K), -1)
        avail = None
        if self.use_actions_mask and avail_actions_list is not None:
            avail = np.stack([np.stack([np.asarray(d[k]) for k in K]) for d in avail_actions_list])
            avail = (avail.reshape(len(obs_list) * len(K), -1) != 0).astype(np.uint8)
        return obs, avail

    def _build_learner(self, *args):
        from ..learners import REGISTRY_Learners
        return REGISTRY_Learners[self.config.learner](*args)

    def finish(self):
        if self.writer is not None:
            self.writer.close()


class OffPolicyMARLAgents(MARLAgents):
    """off_policy_marl.py:17-622."""

    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        super().__init__(config, envs, num_agents, agent_keys, state_space, observation_space, action_space, callback)
        self.on_policy = False
        self.e_greedy = self.start_greedy = config.start_greedy
        self.end_greedy = config.end_greedy
        self.delta_egreedy = (self.start_greedy - self.end_greedy) / config.decay_step_greedy    # per environment step
        self.start_noise = self.end_noise = self.delta_noise = self.noise_scale = None     # discrete actions only
        self.buffer_size, self.batch_size = config.buffer_size, config.batch_size
        if self.world_size > 1:                       # global sizes -> this rank's shard (episodes are independent)
            self.buffer_size //= self.world_size
            self.batch_size //= self.world_size

    def _build_memory(self):
        """off_policy_marl.py:90-107."""
        if not self.use_rnn:
            raise NotImplementedError("hot-path scope: the episode replay of use_rnn=True")
        avail_shape = {k: (self.action_space[k].n,) for k in self.agent_keys} if self.use_actions_mask else None
        return MARL_OffPolicyBuffer_RNN(agent_keys=self.agent_keys,
                                        state_space=self.state_space if self.use_global_state else None,
                                        obs_space=self.observation_space, act_space=self.action_space,
                                        n_envs=self.n_envs, buffer_size=self.buffer_size, batch_size=self.batch_size,
                                        avail_actions_shape=avail_shape, use_actions_mask=self.use_actions_mask,
                                        max_episode_steps=self.episode_length, device=self.device)

    def store_experience(self, obs_list, avail_actions, actions_list, obs_next_list, avail_actions_next, rewards_list,
                         terminals_list, info, **kwargs):
        """off_policy_marl.py:112-159 - per-env dicts -> per-agent [n_envs, ...] arrays -> memory.store."""
        data = {'obs': self._agent_arrays(obs_list), 'actions': self._agent_arrays(actions_list),
                'obs_next': self._agent_arrays(obs_next_list), 'rewards': self._agent_arrays(rewards_list),
                'terminals': self._agent_arrays(terminals_list),
                'agent_mask': self._agent_arrays([d['agent_mask'] for d in info])}
        if self.use_rnn:
            data['episode_steps'] = np.array([d['episode_step'] - 1 for d in info])
        if self.use_global_state:
            data['state'] = np.array(kwargs['state'])
            data['state_next'] = np.array(kwargs['next_state'])
        if self.use_actions_mask:
            data['avail_actions'] = self._agent_arrays(avail_actions)
            data['avail_actions_next'] = self._agent_arrays(avail_actions_next)
        self.memory.store(**data)

    def _build_q_networks(self):
        q_networks = nn.ModuleDict()
        for group_key, group_agents in self.groups.items():
            ref = group_agents[0]
            enc = self._build_agent_feature_encoder(self.config.representation, group_agents, self.observation_space[ref])
            q_networks[group_key] = DiscreteActionValueCritic(
                representation=enc, action_space=self.action_space[ref], critic_hidden_size=self.config.q_hidden_size,
                normalizer=self.normalize_fn, initializer=self.initializer, activation=self.activation,
                device=self.device)
        return q_networks

    def init_rnn_states(self, n_envs):
        return self.model.init_rnn_states(n_envs)

    def init_rnn_states_item(self, i_env, rnn_states=None):
        return self.model.init_rnn_states_item(i_env, rnn_states)

    def _update_explore_factor(self):
        """off_policy_marl.py:198-210."""
        if self.e_greedy > self.end_greedy:
            self.e_greedy = self.start_greedy - self.delta_egreedy * self.current_step
        else:
            self.e_greedy = self.end_greedy

    def exploration(self, batch_size, pi_actions_dict, avail_actions_list=None):
        """off_policy_marl.py:212-255: with probability epsilon the WHOLE vector step acts at random (one draw per call),
        uniformly over each agent's available actions when masks are in use."""
        if np.random.rand() >= self.e_greedy:
            return pi_actions_dict
        if self.use_actions_mask:
            out = []
            for e in range(batch_size):
                d = {}
                for k in self.agent_keys:
                    p = np.asarray(avail_actions_list[e][k], dtype=np.float64)
                    d[k] = int(np.random.choice(len(p), p=p / p.sum()))
                out.append(d)
            return out
        return [{k: self.action_space[k].sample() for k in self.agent_keys} for _ in range(batch_size)]

    @torch.no_grad()
    def get_actions(self, obs_list, avail_actions_list=None, rnn_states=None, test_mode=False, **kwargs):
        """off_policy_marl.py:257-308."""
        batch_size, K = len(obs_list), self.agent_keys
        obs, avail = self._build_inputs(obs_list, avail_actions_list)
        obs_d = torch.from_numpy(obs).to(self.device, non_blocking=True)
        avail_d = torch.from_numpy(avail).to(self.device, non_blocking=True) if avail is not None else None
        actions, _, rnn_new = self.model(observations=obs_d, avail_actions=avail_d, rnn_states=rnn_states)
        acts = actions.reshape(batch_size, len(K)).cpu().numpy()
        actions_list = [{k: int(acts[e, i]) for i, k in enumerate(K)} for e in range(batch_size)]
        if not test_mode:
            actions_list = self.exploration(batch_size, actions_list, avail_actions_list)
        return MARLActionOutput(env_actions=actions_list, rnn_states=rnn_new)

    def train(self, train_steps):
        """off_policy_marl.py:310-354 (the use_rnn branch: whole episodes are collected by run_episodes, then n_epochs
        updates).  Returns the merged training infos."""
        if not self.use_rnn:
            raise NotImplementedError("hot-path scope: use_rnn=True")
        train_info = {}
        step_start = step_last = int(self.current_step)
        n_steps_all = train_steps * self.n_envs
        while step_last - step_start < n_steps_all:
            self.run_episodes(n_episodes=self.n_envs, test_mode=False, close_envs=False)
            if self.current_step >= self.start_training:
                update_info = self.train_epochs(n_epochs=self.n_epochs)
                self.log_infos(update_info, self.current_step)
                train_info.update(update_info)
                self.callback.on_train_epochs_end(self.current_step, model=self.model, memory=self.memory,
                                                  current_episode=self.current_episode, train_steps=train_steps,
                                                  update_info=update_info)
            step_last = int(self.current_step)
        self.callback.on_train_step_end(self.current_step, envs=self.train_envs, model=self.model,
                                        train_steps=train_steps, train_info=train_info)
        return train_info

    def run_episodes(self, n_episodes=1, run_envs=None, test_mode=False, close_envs=True):
        """off_policy_marl.py:426-571."""
        envs = self.train_envs if run_envs is None else run_envs
        num_envs = envs.num_envs
        _current_episode, _current_step, scores, best_score = 0, 0, [], -np.inf
        obs_list, info = envs.reset()
        state = np.array(envs.buf_state, copy=True) if self.use_global_state else None
        avail_actions = list(envs.buf_avail_actions) if self.use_actions_mask else None
        if not test_mode and self.use_rnn:
            self.memory.clear_episodes()
        rnn_states = self.init_rnn_states(num_envs)
        while _current_episode < n_episodes:
            policy_out = self.get_actions(obs_list=obs_list, avail_actions_list=avail_actions, rnn_states=rnn_states,
                                          test_mode=test_mode)
            actions_list, rnn_states = policy_out.env_actions, policy_out.rnn_states
            next_obs_list, rewards_list, terminated_list, truncated, info = envs.step(actions_list)
            next_state = np.array(envs.buf_state, copy=True) if self.use_global_state else None
            next_avail_actions = list(envs.buf_avail_actions) if self.use_actions_mask else None
            if not test_mode:
                self.store_experience(obs_list, avail_actions, actions_list, next_obs_list, next_avail_actions,
                                      rewards_list, terminated_list, info, state=state, next_state=next_state)
            self.callback.on_test_step(envs=envs, model=self.model, test_mode=test_mode, obs=obs_list,
                                       policy_out=policy_out, acts=actions_list, next_obs=next_obs_list,
                                       rewards=rewards_list, terminals=terminated_list, truncations=truncated,
                                       infos=info, state=state, next_state=next_state,
                                       current_train_step=self.current_step, n_episodes=n_episodes,
                                       current_step=_current_step, current_episode=_current_episode)
            obs_list = deepcopy(next_obs_list)
            if self.use_global_state:
                state = deepcopy(next_state)
            if self.use_actions_mask:
                avail_actions = deepcopy(next_avail_actions)
            for i in range(num_envs):
                if all(terminated_list[i].values()) or truncated[i]:
                    _current_episode += 1
                    self._reset_env(envs, i, info, obs_list, state, avail_actions)
                    if self.use_rnn:
                        rnn_states = self.init_rnn_states_item(i_env=i, rnn_states=rnn_states)
                        if not test_mode:
                            terminal_data = {'obs': next_obs_list[i], 'episode_step': info[i]['episode_step']}
                            if self.use_global_state:
                                terminal_data['state'] = next_state[i]
                            if self.use_actions_mask:
                                terminal_data['avail_actions'] = next_avail_actions[i]
                            self.memory.finish_path(i, **terminal_data)
                    episode_score = float(np.mean(itemgetter(*self.agent_keys)(info[i]["episode_score"])))
                    scores.append(episode_score)
                    if test_mode:
                        best_score = max(best_score, episode_score)
                    else:
                        self.current_episode[i] += 1
                        self.current_step += info[i]["episode_step"]
                        self.log_infos({"Train-Results/Episode-Steps": {"env-%d" % i: info[i]["episode_step"]},
                                        "Train-Results/Episode-Rewards": {"env-%d" % i: episode_score}},
                                       self.current_step)
                        self._update_explore_factor()
            _current_step += num_envs
        if test_mode:
            self.log_infos({"Test-Results/Episode-Rewards": float(np.mean(scores)),
                            "Test-Results/Episode-Rewards-Std": float(np.std(scores))}, self.current_step)
            if close_envs:
                envs.close()
        return scores

    def train_epochs(self, n_epochs=1):
        """off_policy_marl.py:573-594."""
        info_train = {}
        for e in range(n_epochs):
            info_train = self.learner.update(self.memory.sample(), sync=(e == n_epochs - 1))
        info_train["epsilon-greedy"] = self.e_greedy
        info_train["noise_scale"] = self.noise_scale
        return info_train

    def test(self, test_episodes, test_envs=None, close_envs=True):
        return self.run_episodes(n_episodes=test_episodes, run_envs=test_envs, test_mode=True, close_envs=close_envs)


class QMIX_Agents(OffPolicyMARLAgents):
    """qmix_agents.py:12-93."""

    def __init__(self, config, envs=None, num_agents=None, agent_keys=None, state_space=None, observation_space=None,
                 action_space=None, callback=None):
        super().__init__(config, envs, num_agents, agent_keys, state_space, observation_space, action_space, callback)
        if self.state_space is None:
            raise ValueError("QMIX mixes on the global state: provide envs or state_space")
        self.use_global_state = True
        # the reference's QMIX divides decay_step_greedy by n_envs (qmix_agents.py); IQL and DCG do not
        self.delta_egreedy = (self.start_greedy - self.end_greedy) / (config.decay_step_greedy / self.n_envs)
        self.model = self._build_model()
        self.memory = self._build_memory()
        self.learner = self._build_learner(self.config, self.agent_grouping, self.model, self.callback)

    def _build_mixer(self):
        return QMIX_Mixer(dim_state=self.state_space.shape[0], dim_hidden=self.config.hidden_dim_mixing_net,
                          dim_hypernet_hidden=self.config.hidden_dim_hyper_net, n_agents=self.n_agents, device=self.device)

    def _build_model(self):
        q_networks = self._build_q_networks()
        mixer = self._build_mixer()
        return MixingQNetwork(grouping=self.agent_grouping, q_networks=q_networks, mixer=mixer, use_rnn=self.use_rnn,
                              device=self.device).to(self.device)


class VDN_Agents(QMIX_Agents):
    """vdn_agents.py: value decomposition with the parameter-free sum mixer; same rollout loop, buffer and learner update
    (the reference's VDN_Learner differs from QMIX_Learner only in not passing the global state to the mixer)."""

    def _build_mixer(self):
        return VDN_mixer()

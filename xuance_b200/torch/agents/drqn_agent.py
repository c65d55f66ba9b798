"""DRQN agent - mirror of xuance/torch/agents/qlearning_family/drqn_agent.py:15-230.

Acting runs the recurrent Q head over one step (K13L with T = 1) from the carried state.  Exploration draws
``np.random.choice(n, n_envs)`` and then ``np.random.rand()`` every step, one coin for all envs, so a seeded agent
reproduces the reference's actions.  ε falls by ``(start - end) / (decay_step_greedy / n_envs)`` per vector step.  An
episode is stored when it terminates or is truncated (its done flags are the terminal flags), and the finished env's
recurrent state is reset."""
from copy import deepcopy

import numpy as np
import torch

from ...common import RecurrentOffPolicyBuffer
from ..rl_models import ActionOutput, DeepRecurrentQNetwork
from .off_policy import OffPolicyAgent


class DRQN_Agent(OffPolicyAgent):
    def __init__(self, config, envs=None, observation_space=None, action_space=None, callback=None):
        super().__init__(config, envs, observation_space, action_space, callback)
        if self.world_size > 1:
            raise NotImplementedError("DRQN: distributed training is not supported (one rank)")
        self.start_greedy, self.end_greedy = config.start_greedy, config.end_greedy
        self.e_greedy = config.start_greedy
        self.delta_egreedy = (self.start_greedy - self.end_greedy) / (config.decay_step_greedy / self.n_envs)
        self.model = self._build_model()
        self.memory = self._build_memory()
        self.learner = self._build_learner(self.config, self.model, self.callback)
        self.lstm = config.rnn == "LSTM"
        self.rnn_states = None

    def _build_memory(self, auxiliary_info_shape=None):
        self.atari = getattr(self.config, "env_name", None) == "Atari"
        return RecurrentOffPolicyBuffer(self.observation_space, self.action_space, auxiliary_info_shape, self.n_envs,
                                        self.buffer_size, self.batch_size, episode_length=self.episode_length,
                                        lookup_length=self.config.lookup_length, device=self.device)

    def _build_model(self):
        rep = self._build_representation(self.config.representation, self.observation_space, self.config)
        return DeepRecurrentQNetwork(representation=rep, recurrent_hidden_size=self.config.recurrent_hidden_size,
                                     recurrent_layer_N=self.config.recurrent_layer_N, dropout=self.config.dropout,
                                     action_space=self.action_space, rnn=self.config.rnn, initializer=self.initializer,
                                     device=self.device, use_distributed_training=self.distributed_training
                                     ).to(self.device)

    @torch.no_grad()
    def get_actions(self, obs, egreedy=0.0, rnn_states=None):
        """drqn_agent.py:69-81."""
        obs = torch.as_tensor(np.asarray(obs), dtype=torch.float32, device=self.device)
        rnn_states_new, out = self.model(obs[:, None], rnn_states)
        random_action = np.random.choice(self.action_space.n, self.n_envs)
        if np.random.rand() < egreedy:
            actions = random_action
        else:
            actions = out.actions.cpu().numpy()
        return ActionOutput(env_actions=actions, rnn_hidden=rnn_states_new)

    def train_epochs(self, n_epochs=1):
        train_info = {}
        for e in range(n_epochs):
            samples = self.memory.sample()
            train_info = self.learner.update(sync=(e == n_epochs - 1), **samples)
        train_info["epsilon-greedy"] = self.e_greedy
        return train_info

    def train(self, train_steps):
        """drqn_agent.py:83-160."""
        train_info = {}
        obs = np.array(self.train_envs.buf_obs, copy=True)
        self.memory.begin(self._process_observation(obs))
        self.rnn_states = self.model.init_rnn_states(self.n_envs)
        for _ in range(train_steps):
            self.obs_rms.update(obs)
            obs = self._process_observation(obs)
            policy_out = self.get_actions(obs, self.e_greedy, self.rnn_states)
            acts = policy_out.env_actions
            self.rnn_states = policy_out.rnn_hidden
            next_obs, rewards, terminals, truncations, infos = self.train_envs.step(acts)
            self.callback.on_train_step(self.current_step, envs=self.train_envs, model=self.model, obs=obs,
                                        policy_out=policy_out, acts=acts, next_obs=next_obs, rewards=rewards,
                                        terminals=terminals, truncations=truncations, infos=infos,
                                        train_steps=train_steps, rnn_states=self.rnn_states)
            if self.current_step > self.start_training and self.current_step % self.training_frequency == 0:
                update_info = self.train_epochs(n_epochs=1)
                self.log_infos(update_info, self.current_step)
                train_info.update(update_info)
            obs = deepcopy(next_obs)
            self.memory.put(self._process_observation(obs), acts, self._process_reward(rewards), terminals)
            reset = []
            for i in range(self.n_envs):
                if terminals[i] or truncations[i]:
                    if self.atari and not truncations[i]:
                        continue
                    self.rnn_states = self.model.init_rnn_states_item(self.rnn_states, i)
                    self.current_episode[i] += 1
                    episode_info = {f"Episode-Steps/rank_{self.rank}": {f"env-{i}": infos[i]["episode_step"]},
                                    f"Train-Episode-Rewards/rank_{self.rank}": {f"env-{i}": infos[i]["episode_score"]}}
                    self.log_infos(episode_info, self.current_step)
                    train_info.update(episode_info)
                    self.memory.store(i)
                    obs[i] = infos[i]["reset_obs"]
                    self.train_envs.buf_obs[i] = obs[i]
                    reset.append(i)
                    self.callback.on_train_episode_info(envs=self.train_envs, model=self.model, env_id=i,
                                                        memory=self.memory, infos=infos, rank=self.rank,
                                                        use_wandb=False, current_step=self.current_step,
                                                        current_episode=self.current_episode, train_steps=train_steps)
            if reset:
                self.memory.begin(self._process_observation(obs), reset)
            self.current_step += self.n_envs
            if self.e_greedy > self.end_greedy:
                self.e_greedy = self.e_greedy - self.delta_egreedy
            self.callback.on_train_step_end(self.current_step, envs=self.train_envs, model=self.model,
                                            train_steps=train_steps, train_info=train_info)
        return train_info

    def test(self, test_episodes=1, test_envs=None, close_envs=True):
        """drqn_agent.py:162-230 (no video): greedy actions from a carried state that resets per finished env."""
        envs = test_envs or self.train_envs
        obs, _ = envs.reset()
        scores = []
        rnn_states = self.model.init_rnn_states(envs.num_envs)
        while len(scores) < test_episodes:
            self.obs_rms.update(obs)
            out = self.get_actions(self._process_observation(obs), egreedy=0.0, rnn_states=rnn_states)
            rnn_states = out.rnn_hidden
            next_obs, rewards, terminals, truncations, infos = envs.step(out.env_actions)
            obs = deepcopy(next_obs)
            for i in range(envs.num_envs):
                if terminals[i] or truncations[i]:
                    if self.atari and not truncations[i]:
                        continue
                    obs[i] = infos[i]["reset_obs"]
                    rnn_states = self.model.init_rnn_states_item(rnn_states, i)
                    scores.append(float(infos[i]["episode_score"]))
        if close_envs and test_envs is not None:
            envs.close()
        return scores[:test_episodes]

"""Uniform replay with the reference's `Replay` API (replay_memory.py:4-80), device-resident.

  Replay(max_size, env, n_steps=1, gamma=0.99).add(state, action, reward, next_state, done)
  .sample(batch_size) -> (states, actions, rewards, next_states, terminates), all float64,
                         shaped (batch_size, -1) like the reference (replay_memory.py:75-80)

Sampling positions come from `random.sample(range(len), B)` -- the same positions
`random.sample(self.buffer, B)` picks for the same generator state -- and the rows are gathered
on the GPU.
"""
import random

import numpy as np

from .obs_norm import make_obs_normalizer
from .prioritized_replay_memory import _DeviceReplay


class Replay(object):
    def __init__(self, max_size, env, n_steps=1, gamma=0.99, obs_dim=None, act_dim=None, device=None, obs_norm=None,
                 nstep_tails=False):
        self.capacity = max_size
        self.env = env
        self.n_steps = n_steps
        self.gamma = gamma
        # obs_norm: None / False, True, {"clip": c, "eps": e} or an ObsNormalizer that every insert updates (obs_norm.py);
        # nstep_tails: add_steps also stores the last n_steps - 1 starts of every episode (ReplayBuffer.add_steps)
        self._store = _DeviceReplay(max_size, 1.0, False, obs_dim, act_dim, device,
                                    make_obs_normalizer(obs_norm, obs_dim, device), nstep_tails)

    @property
    def obs_normalizer(self):
        return self._store.obs_norm

    def __len__(self):
        return len(self._store)

    @property
    def position(self):
        return (self._store._next_idx + self._store._n_staged) % self._store.size

    def add(self, state, action, reward, next_state, done):
        self._store.add(state, action, reward, next_state, done)

    def add_batch(self, state, action, reward, next_state, done):
        if isinstance(state, np.ndarray):
            self._store.add_batch_host(state, action, reward, next_state, done)
        else:
            self._store.add_batch(state, action, reward, next_state, done)

    def add_episode(self, states, actions, rewards, next_states, dones):
        """One episode of consecutive steps; the n-step return (self.n_steps, self.gamma) is accumulated on the device
        at insert -- the arithmetic of initialize() below / replay_memory.py:38-45."""
        return self._store.add_episode_nstep(states, actions, rewards, next_states, dones, self.n_steps, self.gamma)

    def add_steps(self, states, actions, rewards, next_states, terminated, truncated=None, n_steps=None, gamma=None):
        """One vector step of E environments with the n-step windows on the device, at this Replay's n_steps / gamma
        (ReplayBuffer.add_steps has the semantics).  n_steps / gamma, when given, must equal the Replay's.  Returns the
        number of rows inserted."""
        if (n_steps is not None and n_steps != self.n_steps) or (gamma is not None and float(gamma) != float(self.gamma)):
            raise ValueError("Replay.add_steps: this Replay forms %d-step returns at gamma=%r, got n_steps=%r, gamma=%r"
                             % (self.n_steps, self.gamma, n_steps, gamma))
        return self._store.add_steps(states, actions, rewards, next_states, terminated, truncated, self.n_steps, self.gamma)

    def drop_steps(self):
        """Discard the pending n-step windows of add_steps."""
        self._store.drop_steps()

    def add_goal_steps(self, obs, desired_goal, action, reward, obs_next, achieved_goal_next, terminated, truncated=None,
                       her_ratio=0.8, threshold=0.05, her_action="reference", max_episode_steps=50, seed=0):
        """One vector step of E goal-conditioned environments with hindsight relabelling on the device
        (ReplayBuffer.add_goal_steps has the semantics).  One-step rows: this Replay's n_steps is not applied.  Returns
        the number of rows inserted."""
        return self._store.add_goal_steps(obs, desired_goal, action, reward, obs_next, achieved_goal_next, terminated,
                                          truncated, her_ratio, threshold, her_action, max_episode_steps, seed)

    def flush_goal_steps(self):
        """Insert the episodes of add_goal_steps that have ended, without taking a step."""
        return self._store.flush_goal_steps()

    def drop_goal_steps(self):
        """Discard the pending episodes of add_goal_steps."""
        self._store.drop_goal_steps()

    def initialize(self, init_length):
        """Random-policy filler with n-step return accumulation at insert time (replay_memory.py:21-59).  Needs a
        gym-style `env`.  The rollout is host glue; every finished (or cut-off) episode goes to the device in one
        `add_episode` call, which forms the n-step transitions there.  The reference stops the moment the buffer holds
        `init_length` transitions, possibly mid-episode: the last episode is truncated to the steps it had taken."""
        env = self.env
        while len(self) < init_length:
            state = env.reset()
            states, actions, rewards, nexts, dones = [], [], [], [], []
            have = len(self)
            while True:
                action = np.random.uniform(-1.0, 1.0, size=env.action_space.shape)
                next_state, reward, done, _ = env.step(action)
                states.append(np.asarray(state).reshape(-1)); actions.append(action); rewards.append(reward)
                nexts.append(np.asarray(next_state).reshape(-1)); dones.append(done)
                added = max(0, len(rewards) - self.n_steps + 1)               # transitions this episode contributes so far
                if have + added >= init_length or done:
                    break
                state = next_state
            if len(rewards) >= self.n_steps:
                self.add_episode(np.stack(states), np.stack(actions), np.asarray(rewards, dtype=np.float64), np.stack(nexts),
                                 np.asarray(dones))

    def sample_positions(self, batch_size):
        return random.sample(range(len(self)), batch_size)                 # replay_memory.py:67

    def sample(self, batch_size, positions=None):
        if positions is None:
            positions = self.sample_positions(batch_size)
        o = self._store.gather(positions)
        f64 = np.float64
        B = batch_size
        return (o["s"].cpu().numpy().astype(f64).reshape(B, -1), o["a"].cpu().numpy().astype(f64).reshape(B, -1),
                o["r"].cpu().numpy().astype(f64).reshape(B, -1), o["s2"].cpu().numpy().astype(f64).reshape(B, -1),
                o["d"].cpu().numpy().astype(f64).reshape(B, -1))

"""TEST INFRASTRUCTURE -- the classic-control tasks of surreal_b200.env.classic in float64 numpy: CartPole-v1 and
Pendulum-v1 with gym's classic_control dynamics, their episode cap, auto-reset and Philox reset draws.

These tasks have no counterpart in the reference, which reaches them through gym; this module defines the semantics the
device kernels implement (surreal_b200/csrc/env.cu).  Physics runs in float64 on the given (float32) states;
the reset draws are exact: the kernels form them in float32 with the same roundings.

``ClassicRef`` is also a batched host env (attributes N, D, A; numpy reset / step), so the host-env path of the agents
can be driven with the same tasks."""
import math

import numpy as np

from oracle.philox import philox4x32_10

CARTPOLE, PENDULUM = 0, 1                   # task ids of this module
CLASSIC_KEY = 0xD6E8FEB86659FD93            # the reset stream's key: env seed ^ CLASSIC_KEY
REGISTERED_LIMIT = {CARTPOLE: 500, PENDULUM: 200}
DIMS = {CARTPOLE: (4, 4, 2), PENDULUM: (2, 3, 1)}      # state, observation, action widths

# CartPole-v1
GRAVITY, MASS_CART, MASS_POLE, LENGTH, FORCE_MAG, TAU = 9.8, 1.0, 0.1, 0.5, 10.0, 0.02
TOTAL_MASS = MASS_CART + MASS_POLE
POLEMASS_LENGTH = MASS_POLE * LENGTH
# the state is float32, so the termination thresholds are the float32 values of 2.4 and 12 * 2 pi / 360
X_THRESHOLD = float(np.float32(2.4))
THETA_THRESHOLD = float(np.float32(12 * 2 * math.pi / 360))

# Pendulum-v1
G, M, L, DT, MAX_SPEED, MAX_TORQUE = 10.0, 1.0, 1.0, 0.05, 8.0, 2.0


def reset_uniforms(seed, episode, actor_ids):
    """The four uniforms of each actor's reset draw -> float32 [n, 4]: Philox4x32-10 keyed (seed ^ CLASSIC_KEY,
    counter = (episode index, actor)), u_k = (word_k >> 8) * 2^-24 (exact in float32)."""
    ids = np.asarray(actor_ids, dtype=np.uint64)
    ep = np.broadcast_to(np.asarray(episode, dtype=np.uint64), ids.shape)
    words = philox4x32_10(np.uint64(int(seed) ^ CLASSIC_KEY), ep, ids)
    return np.stack([(w >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24) for w in words], axis=1)


def _draw(u, lo, width):
    """lo + width * u in float32, rounded after the product and after the sum."""
    return (np.float32(width) * u).astype(np.float32) + np.float32(lo)


def reset_state(task, seed, episode, actor_ids):
    """Start state of episode ``episode`` (scalar or per actor) of the given actors -> float32 [n, S].
    CartPole: each component uniform in [-0.05, 0.05]; Pendulum: theta in [-pi, pi], theta_dot in [-1, 1]."""
    u = reset_uniforms(seed, episode, actor_ids)
    if task == CARTPOLE:
        return _draw(u, -0.05, 0.1).astype(np.float32)
    return np.stack([_draw(u[:, 0], -math.pi, 2 * math.pi), _draw(u[:, 1], -1.0, 2.0)], axis=1).astype(np.float32)


def observe(task, s):
    """Observation of states s [n, S] -> float64 [n, D]."""
    s = np.asarray(s, dtype=np.float64)
    if task == CARTPOLE:
        return s.copy()
    return np.stack([np.cos(s[:, 0]), np.sin(s[:, 0]), s[:, 1]], axis=1)


def angle_normalize(x):
    """((x + pi) mod 2 pi) - pi, Python's mod (the sign of the divisor): both pi and -pi map to -pi."""
    return np.mod(np.asarray(x, dtype=np.float64) + math.pi, 2 * math.pi) - math.pi


def cartpole_terminal(s):
    s = np.asarray(s, dtype=np.float64)
    return (s[:, 0] < -X_THRESHOLD) | (s[:, 0] > X_THRESHOLD) | (s[:, 2] < -THETA_THRESHOLD) | (s[:, 2] > THETA_THRESHOLD)


def cartpole_step(s, push_right):
    """One explicit-Euler step -> (successor [n, 4] float64, reward [n], terminal [n] bool)."""
    x, x_dot, th, th_dot = np.asarray(s, dtype=np.float64).T
    force = np.where(np.asarray(push_right, dtype=bool), FORCE_MAG, -FORCE_MAG)
    cs, sn = np.cos(th), np.sin(th)
    temp = (force + POLEMASS_LENGTH * th_dot ** 2 * sn) / TOTAL_MASS
    thacc = (GRAVITY * sn - cs * temp) / (LENGTH * (4.0 / 3.0 - MASS_POLE * cs ** 2 / TOTAL_MASS))
    xacc = temp - POLEMASS_LENGTH * thacc * cs / TOTAL_MASS
    nxt = np.stack([x + TAU * x_dot, x_dot + TAU * xacc, th + TAU * th_dot, th_dot + TAU * thacc], axis=1)
    return nxt, np.ones(len(nxt)), cartpole_terminal(nxt)


def pendulum_step(s, a):
    """One step with actions a [n] (or [n, 1]) in [-1, 1] -> (successor [n, 2] float64, reward [n], terminal [n])."""
    th, th_dot = np.asarray(s, dtype=np.float64).T
    u = MAX_TORQUE * np.clip(np.asarray(a, dtype=np.float64).reshape(-1), -1.0, 1.0)
    cost = angle_normalize(th) ** 2 + 0.1 * th_dot ** 2 + 0.001 * u ** 2
    new_th_dot = np.clip(th_dot + (3 * G / (2 * L) * np.sin(th) + 3.0 / (M * L ** 2) * u) * DT, -MAX_SPEED, MAX_SPEED)
    nxt = np.stack([th + new_th_dot * DT, new_th_dot], axis=1)
    return nxt, -cost, np.zeros(len(nxt), dtype=bool)


def push_right(action, n):
    """CartPole's action as 'index 1': int indices [n], or one-hot rows [n, 2] (row[1] > row[0])."""
    a = np.asarray(action)
    if a.ndim == 2:
        return a[:, 1] > a[:, 0]
    return a.reshape(n) == 1


def physics_step(task, s, action):
    if task == CARTPOLE:
        return cartpole_step(s, push_right(action, len(s)))
    return pendulum_step(s, action)


class ClassicRef:
    """N actors of one task.  Each actor has a state, an episode step and an episode index; done = terminal or the
    episode step reaching the cap (``limit_episode_length`` > 0, else the registered limit); done actors start their
    next episode in the same step.  The state is kept in float64 (the physics of the successive steps is not rounded
    to float32), so long trajectories drift from the kernels' float32 ones; tests compare one step at a time."""

    def __init__(self, task, N, limit_episode_length=0, seed=0):
        self.task, self.N, self.seed = task, int(N), int(seed)
        self.S, self.D, self.A = DIMS[task]
        self.max_steps = int(limit_episode_length) if int(limit_episode_length) > 0 else REGISTERED_LIMIT[task]
        self.state = np.zeros((self.N, self.S))
        self.ep_step = np.zeros(self.N, dtype=np.int64)
        self.episode = np.zeros(self.N, dtype=np.int64)

    def _obs(self, s):
        return {'low_dim': {'flat_inputs': observe(self.task, s).astype(np.float32)}}

    def reset(self):
        self.ep_step[:] = 0
        self.episode[:] = 0
        self.state = reset_state(self.task, self.seed, 0, np.arange(self.N)).astype(np.float64)
        return self._obs(self.state), {}

    def step(self, action):
        """-> (obs, reward float32 [N], done float32 [N], {'obs_next': ...}) as the device env returns them."""
        nxt, rew, term = physics_step(self.task, self.state, action)
        self.ep_step += 1
        done = term | (self.ep_step >= self.max_steps)
        obs_next = observe(self.task, nxt).astype(np.float32)
        s = nxt.copy()
        if done.any():
            ids = np.nonzero(done)[0]
            self.episode[ids] += 1
            s[ids] = reset_state(self.task, self.seed, self.episode[ids], ids)
            self.ep_step[ids] = 0
        self.state = s
        return self._obs(s), rew.astype(np.float32), done.astype(np.float32), {'obs_next': obs_next}

"""Classic-control tasks as batched, device-resident envs: CartPole-v1 and Pendulum-v1 with gym's dynamics, one CUDA
thread per actor (csrc/env.cu; the float64 statement of both tasks is tests/classic_ref.py).  They have
SyntheticEnv's interface, so every agent and engine that runs the synthetic env runs them, and unlike it they have a
known solution: a policy that learns them shows that training works end to end.

The episode cap is MaxStepWrapper's (surreal/env/wrapper.py:142-163), as in SyntheticEnv: ``limit_episode_length``
when > 0, else the task's registered limit (CartPole-v1 500, Pendulum-v1 200).  Reaching it sets done = 1 and is
treated as terminal.  Done actors auto-reset inside the same launch, from Philox draws keyed by (seed, actor) with the
actor's episode index as the counter, so the seed fixes the whole trajectory for a given action stream."""
import ctypes as C

import torch

from .. import _lib
from .._lib import check
from ..ops import _stream
from .base import LowDimEnv


class _ClassicEnv(LowDimEnv):
    S = MAX_STEPS = ACTION_TYPE = None
    NAME = ''

    def __init__(self, num_envs, limit_episode_length=0, seed=0, device=None):
        lim = int(limit_episode_length)
        super().__init__(num_envs, self.D, self.A, lim if lim > 0 else self.MAX_STEPS, seed, device)
        f = lambda *s: torch.zeros(*s, device=self.device)  # noqa: E731
        self.state = f(self.N, self.S)
        self.obs = f(self.N, self.D)
        self.obs_next = f(self.N, self.D)
        self.episode = torch.zeros(self.N, dtype=torch.int32, device=self.device)
        self._describe(self.seed, obs=self.obs, episode=self.episode)

    def action_spec(self):
        return {'dim': (self.A,), 'type': self.ACTION_TYPE}

    def reset(self):
        check(_lib.lib().sb200_env_reset_f32(C.byref(self.desc), _stream()), 'sb200_env_reset_f32')
        return self._obs(self.obs), {}


class CartPoleEnv(_ClassicEnv):
    """CartPole-v1: observation (x, x_dot, theta, theta_dot); two discrete actions as one-hot rows [N, 2] (index 1 pushes
    right); reward 1 per step; terminal when |x| > 2.4 or |theta| > 12 degrees."""
    KIND, S, D, A, MAX_STEPS, ACTION_TYPE = _lib.ENV_CARTPOLE, 4, 4, 2, 500, 'discrete'
    NAME = 'CartPole-v1'


class PendulumEnv(_ClassicEnv):
    """Pendulum-v1: observation (cos theta, sin theta, theta_dot); one continuous action in [-1, 1], scaled to the torque
    2a; reward -(theta^2 + 0.1 theta_dot^2 + 0.001 torque^2); never terminal."""
    KIND, S, D, A, MAX_STEPS, ACTION_TYPE = _lib.ENV_PENDULUM, 2, 3, 1, 200, 'continuous'
    NAME = 'Pendulum-v1'


CLASSIC_ENVS = {cls.NAME: cls for cls in (CartPoleEnv, PendulumEnv)}
CLASSIC_PREFIX = 'classic:'


def classic_env_class(name):
    """The env class of a ``classic:<task>`` env name, None for any other name; an unknown task raises."""
    name = str(name)
    if not name.startswith(CLASSIC_PREFIX):
        return None
    task = name[len(CLASSIC_PREFIX):]
    if task not in CLASSIC_ENVS:
        raise ValueError('unknown classic-control task %r: one of %s' % (task, ', '.join(sorted(CLASSIC_ENVS))))
    return CLASSIC_ENVS[task]


def make_classic_env(env_config, num_envs):
    """The env of a ``classic:<task>`` env config, or None for any other env name."""
    cls = classic_env_class(env_config.env_name if 'env_name' in env_config else '')
    if cls is None:
        return None
    return cls(num_envs, env_config.limit_episode_length, seed=int(env_config.seed) if 'seed' in env_config else 0)

"""Base of the batched, device-resident envs (csrc/env.cu): the synthetic envs of the benchmark configs and the
classic-control tasks.  Every buffer an env owns is allocated once, at a fixed address, so its sb200_env descriptor is
filled once in __init__ and a step is one C call with no host logic (CUDA-graph capturable)."""
import ctypes as C

import torch

from .. import _lib
from .._lib import check
from ..ops import _ptr, _stream


class DeviceEnv:
    """N actors stepped on the device by sb200_env_step_f32.  A subclass sets KIND, allocates its own buffers after
    this __init__ (at least ``state`` and ``obs_next``) and then calls _describe."""
    metadata = {}
    graph_safe = True          # every buffer at a fixed address, no host logic inside step()
    KIND = None

    def __init__(self, num_envs, obs_dim, action_dim, max_steps, seed, device):
        if not torch.cuda.is_available():
            raise RuntimeError('%s is device-resident: a CUDA device is required' % type(self).__name__)
        self.device = torch.device(device if device is not None else ('cuda:%d' % torch.cuda.current_device()))
        self.N, self.D, self.A = int(num_envs), int(obs_dim), int(action_dim)
        self.max_steps = int(max_steps)
        self.seed = int(seed)
        self.ep_step = torch.zeros(self.N, dtype=torch.int32, device=self.device)
        self.reward = torch.zeros(self.N, device=self.device)
        self.done = torch.zeros(self.N, device=self.device)
        self.step_counter = torch.zeros(1, dtype=torch.int64, device=self.device)   # the agents' Philox step counter

    def _describe(self, key, obs=None, **buffers):
        """Fills the descriptor: ``key`` is the seed the kernels draw with, ``obs`` what the actors observe next where
        that is not the state, ``buffers`` the kind's other tensors (WsT / WaT, episode)."""
        self._observed = self.state if obs is None else obs
        ptrs = {k: v.data_ptr() for k, v in buffers.items()}
        if obs is not None:
            ptrs['obs'] = obs.data_ptr()
        self.desc = _lib.Env(kind=self.KIND, N=self.N, D=self.D, A=self.A, max_steps=self.max_steps, seed=key,
                             state=self.state.data_ptr(), ep_step=self.ep_step.data_ptr(),
                             step_counter=self.step_counter.data_ptr(), obs_next=self.obs_next.data_ptr(),
                             reward=self.reward.data_ptr(), done=self.done.data_ptr(), **ptrs)

    def action_spec(self):
        return {'dim': (self.A,), 'type': 'continuous'}

    def _action(self, action):
        if isinstance(action, tuple):            # QAgent.act: (one-hot rows, indices)
            action = action[0]
        # one actor's action may come without the batch dimension, as the agents return it for a single actor
        shapes = [(self.N, self.A)] + ([(self.A,)] if self.N == 1 else [])
        if not (isinstance(action, torch.Tensor) and tuple(action.shape) in shapes and action.is_cuda and
                action.dtype == torch.float32 and action.is_contiguous()):
            raise ValueError('%s.step takes a contiguous float32 CUDA tensor [%d, %d]' % (type(self).__name__, self.N,
                                                                                          self.A))
        return action

    def _step(self, action, windows):
        check(_lib.lib().sb200_env_step_f32(C.byref(self.desc), _ptr(self._action(action)), windows, _stream()),
              'sb200_env_step_f32')

    def step(self, action):
        """action: [N, A] CUDA tensor (or QAgent.act's (one-hot rows, indices) pair).  Returns (obs, reward, done, info):
        obs is what every actor observes NEXT (already reset where done); ``info['obs_next']`` is the true successor
        (terminal where done)."""
        self._step(action, None)
        return self._result()

    def close(self):
        pass


class LowDimEnv(DeviceEnv):
    """A DeviceEnv whose observations are flat float rows [N, D]; its step can be fused with the window commit."""

    def observation_spec(self):
        return {'low_dim': {'flat_inputs': (self.D,)}}

    def _obs(self, x):
        return {'low_dim': {'flat_inputs': x}}

    def _result(self):
        return self._obs(self._observed), self.reward, self.done, {'obs_next': self.obs_next}

    def step_and_commit_window(self, action, w):
        """step() fused with the commit half of ExpSenderWrapperMultiStepMovingWindowWithInfo.step (``w``), for
        steps whose replay slots the sampling kernel has already assigned."""
        self._step(action, C.byref(w.windows))
        return self._result()

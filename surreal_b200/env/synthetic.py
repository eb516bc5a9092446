"""Batched, device-resident synthetic environment of the benchmark configs (SURVEY.md §8d, cfg 2/3/5):

    s' = tanh(Ws s + Wa a) + 0.01 xi,   r = -|s|^2 / D + 0.1 xi',   Ws, Wa ~ N(0, 1/sqrt(D)),  s0 ~ N(0,1)

with the episode cap of MaxStepWrapper (surreal/env/wrapper.py:142-163) folded in: ``done`` when an
actor's episode reaches ``limit_episode_length``; done actors auto-reset.  All N actors advance with ONE
kernel launch and every tensor stays in HBM.  The gym / MuJoCo / robosuite adapters of surreal/env are out
of scope (SURVEY §2 row 6); an external CPU env can still drive ``agent.act`` with numpy observations."""
import ctypes as C

import torch

from .. import _lib
from .._lib import check
from ..ops import _stream


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class SyntheticEnv:
    metadata = {}
    graph_safe = True          # obs IS the state buffer: fixed address, no host logic inside step()

    def __init__(self, num_envs, obs_dim=64, action_dim=8, limit_episode_length=200, seed=0, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError('SyntheticEnv is device-resident: a CUDA device is required')
        self.device = torch.device(device if device is not None else ('cuda:%d' % torch.cuda.current_device()))
        self.N, self.D, self.A = num_envs, obs_dim, action_dim
        self.max_steps = int(limit_episode_length)
        self.seed = int(seed)
        g = torch.Generator().manual_seed(self.seed)
        scale = 1.0 / (obs_dim ** 0.5)
        self.Ws = (torch.randn(obs_dim, obs_dim, generator=g) * scale).to(self.device)
        self.Wa = (torch.randn(obs_dim, action_dim, generator=g) * scale).to(self.device)
        self.WsT, self.WaT = self.Ws.t().contiguous(), self.Wa.t().contiguous()     # kernel layout (k-major)
        self._g = torch.Generator().manual_seed(self.seed + 1)
        self.state = torch.zeros(num_envs, obs_dim, device=self.device)
        self.ep_step = torch.zeros(num_envs, dtype=torch.int32, device=self.device)
        self.obs_next = torch.zeros(num_envs, obs_dim, device=self.device)
        self.reward = torch.zeros(num_envs, device=self.device)
        self.done = torch.zeros(num_envs, device=self.device)
        self.step_counter = torch.zeros(1, dtype=torch.int64, device=self.device)   # shared Philox counter
        self._own_counter = True

    def observation_spec(self):
        return {'low_dim': {'flat_inputs': (self.D,)}}

    def action_spec(self):
        return {'dim': (self.A,), 'type': 'continuous'}

    def reset(self):
        self.state.copy_(torch.randn(self.N, self.D, generator=self._g).to(self.device))
        self.ep_step.zero_()
        return {'low_dim': {'flat_inputs': self.state}}, {}

    def step(self, action):
        """action: [N, A] CUDA tensor.  Returns (obs, reward, done, info): obs is what every actor observes NEXT
        (already reset where done); ``info['obs_next']`` is the true successor (terminal where done)."""
        if isinstance(action, tuple):
            action = action[0]
        check(_lib.lib().sb200_synth_env_step_f32(
            _p(self.state), _p(action), _p(self.WsT), _p(self.WaT), self.N, self.D, self.A, self.max_steps,
            _p(self.ep_step), self.seed + 7, _p(self.step_counter), _p(self.obs_next), _p(self.reward), _p(self.done),
            _stream()), 'sb200_synth_env_step_f32')
        return {'low_dim': {'flat_inputs': self.state}}, self.reward, self.done, {'obs_next': self.obs_next}

    def step_and_commit_window(self, action, w):
        """step() fused with the commit half of ExpSenderWrapperMultiStepMovingWindowWithInfo.step (``w``), for
        steps whose replay slots the sampling kernel has already assigned."""
        check(_lib.lib().sb200_synth_env_window_step_f32(
            _p(self.state), _p(action), _p(self.WsT), _p(self.WaT), self.N, self.D, self.A, self.max_steps,
            _p(self.ep_step), self.seed + 7, _p(self.step_counter), _p(self.obs_next), _p(self.reward), _p(self.done),
            C.byref(w.windows), _stream()), 'sb200_synth_env_window_step_f32')
        return {'low_dim': {'flat_inputs': self.state}}, self.reward, self.done, {'obs_next': self.obs_next}

    def close(self):
        pass


class DiscreteSyntheticEnv(SyntheticEnv):
    """SyntheticEnv with ``n_actions`` discrete actions: the same arithmetic driven by one-hot rows a = e_k, so the action
    term Wa a is column k of Wa [D][n_actions].  step() takes the one-hot rows [N, n_actions] (or QAgent.act's
    (one-hot rows, indices) pair)."""

    def __init__(self, num_envs, obs_dim=64, n_actions=18, limit_episode_length=200, seed=0, device=None):
        super().__init__(num_envs, obs_dim, n_actions, limit_episode_length, seed, device)
        self.n_actions = int(n_actions)

    def action_spec(self):
        return {'dim': (self.n_actions,), 'type': 'discrete'}


class SyntheticPixelEnv:
    """Batched device-resident PIXEL env of BASELINE configs[3] (SURVEY §8d cfg 4): every step each actor observes a fresh
    uint8 frame [C, H, W] of uniform random bytes; reward = -mean(a^2) + 0.1 xi; episodes end at ``limit_episode_length``.
    The staging / replay kernels see a frame as C*H*W/4 opaque 32-bit words (``D``), so frames stay uint8 in HBM."""
    metadata = {}
    graph_safe = True

    def __init__(self, num_envs, frame_shape=(4, 84, 84), action_dim=8, limit_episode_length=200, seed=0, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError('SyntheticPixelEnv is device-resident: a CUDA device is required')
        self.device = torch.device(device if device is not None else ('cuda:%d' % torch.cuda.current_device()))
        self.N, self.A = num_envs, action_dim
        self.frame_shape = tuple(int(v) for v in frame_shape)
        self.frame_bytes = 1
        for v in self.frame_shape:
            self.frame_bytes *= v
        assert self.frame_bytes % 16 == 0, 'C*H*W must be a multiple of 16 bytes'
        self.D = self.frame_bytes // 4
        self.max_steps = int(limit_episode_length)
        self.seed = int(seed)
        self._g = torch.Generator().manual_seed(self.seed + 1)
        self.state = torch.zeros(num_envs, self.frame_bytes, dtype=torch.uint8, device=self.device)
        self.obs_next = torch.zeros_like(self.state)
        self.ep_step = torch.zeros(num_envs, dtype=torch.int32, device=self.device)
        self.reward = torch.zeros(num_envs, device=self.device)
        self.done = torch.zeros(num_envs, device=self.device)
        self.step_counter = torch.zeros(1, dtype=torch.int64, device=self.device)

    def _obs(self, frames):
        return {'pixel': {'camera0': frames.view(self.N, *self.frame_shape)}}

    def observation_spec(self):
        return {'pixel': {'camera0': self.frame_shape}}

    def action_spec(self):
        return {'dim': (self.A,), 'type': 'continuous'}

    def reset(self):
        self.state.copy_(torch.randint(0, 256, (self.N, self.frame_bytes), generator=self._g, dtype=torch.uint8).to(self.device))
        self.ep_step.zero_()
        return self._obs(self.state), {}

    def step(self, action):
        if isinstance(action, tuple):
            action = action[0]
        check(_lib.lib().sb200_synth_pixel_env_step_u8(
            _p(self.state), _p(action), self.N, self.frame_bytes, self.A, self.max_steps, _p(self.ep_step), self.seed + 7,
            _p(self.step_counter), _p(self.obs_next), _p(self.reward), _p(self.done), _stream()), 'sb200_synth_pixel_env_step_u8')
        return self._obs(self.state), self.reward, self.done, {'obs_next': self._obs(self.obs_next)}

    def close(self):
        pass

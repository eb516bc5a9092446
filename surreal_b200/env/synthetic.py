"""Batched, device-resident synthetic environment of the benchmark configs (SURVEY.md §8d, cfg 2/3/5):

    s' = tanh(Ws s + Wa a) + 0.01 xi,   r = -|s|^2 / D + 0.1 xi',   Ws, Wa ~ N(0, 1/sqrt(D)),  s0 ~ N(0,1)

with the episode cap of MaxStepWrapper (surreal/env/wrapper.py:142-163) folded in: ``done`` when an
actor's episode reaches ``limit_episode_length``; done actors auto-reset.  All N actors advance with ONE
kernel launch and every tensor stays in HBM.  The gym / MuJoCo / robosuite adapters of surreal/env are out
of scope (SURVEY §2 row 6); an external CPU env can still drive ``agent.act`` with numpy observations."""
import torch

from .. import _lib
from .base import DeviceEnv, LowDimEnv

NOISE_KEY_OFFSET = 7       # the synthetic envs' kernels draw their noise keyed by seed + 7


class SyntheticEnv(LowDimEnv):
    KIND = _lib.ENV_SYNTH

    def __init__(self, num_envs, obs_dim=64, action_dim=8, limit_episode_length=200, seed=0, device=None):
        super().__init__(num_envs, obs_dim, action_dim, limit_episode_length, seed, device)
        g = torch.Generator().manual_seed(self.seed)
        scale = 1.0 / (obs_dim ** 0.5)
        self.Ws = (torch.randn(obs_dim, obs_dim, generator=g) * scale).to(self.device)
        self.Wa = (torch.randn(obs_dim, action_dim, generator=g) * scale).to(self.device)
        self.WsT, self.WaT = self.Ws.t().contiguous(), self.Wa.t().contiguous()     # kernel layout (k-major)
        self._g = torch.Generator().manual_seed(self.seed + 1)
        self.state = torch.zeros(num_envs, obs_dim, device=self.device)             # obs IS the state buffer
        self.obs_next = torch.zeros(num_envs, obs_dim, device=self.device)
        self._describe(self.seed + NOISE_KEY_OFFSET, WsT=self.WsT, WaT=self.WaT)

    def reset(self):
        self.state.copy_(torch.randn(self.N, self.D, generator=self._g).to(self.device))
        self.ep_step.zero_()
        return self._obs(self.state), {}


class DiscreteSyntheticEnv(SyntheticEnv):
    """SyntheticEnv with ``n_actions`` discrete actions: the same arithmetic driven by one-hot rows a = e_k, so the action
    term Wa a is column k of Wa [D][n_actions].  step() takes the one-hot rows [N, n_actions] (or QAgent.act's
    (one-hot rows, indices) pair)."""

    def __init__(self, num_envs, obs_dim=64, n_actions=18, limit_episode_length=200, seed=0, device=None):
        super().__init__(num_envs, obs_dim, n_actions, limit_episode_length, seed, device)
        self.n_actions = int(n_actions)

    def action_spec(self):
        return {'dim': (self.n_actions,), 'type': 'discrete'}


class SyntheticPixelEnv(DeviceEnv):
    """Batched device-resident PIXEL env of BASELINE configs[3] (SURVEY §8d cfg 4): every step each actor observes a fresh
    uint8 frame [C, H, W] of uniform random bytes; reward = -mean(a^2) + 0.1 xi; episodes end at ``limit_episode_length``.
    The staging / replay kernels see a frame as C*H*W/4 opaque 32-bit words (``D``), so frames stay uint8 in HBM.  Its
    rows are too wide for the fused window commit, so it has no step_and_commit_window."""
    KIND = _lib.ENV_SYNTH_PIXEL

    def __init__(self, num_envs, frame_shape=(4, 84, 84), action_dim=8, limit_episode_length=200, seed=0, device=None):
        self.frame_shape = tuple(int(v) for v in frame_shape)
        self.frame_bytes = 1
        for v in self.frame_shape:
            self.frame_bytes *= v
        assert self.frame_bytes % 16 == 0, 'C*H*W must be a multiple of 16 bytes'
        super().__init__(num_envs, self.frame_bytes // 4, action_dim, limit_episode_length, seed, device)
        self._g = torch.Generator().manual_seed(self.seed + 1)
        self.state = torch.zeros(num_envs, self.frame_bytes, dtype=torch.uint8, device=self.device)
        self.obs_next = torch.zeros_like(self.state)
        self._describe(self.seed + NOISE_KEY_OFFSET)

    def _obs(self, frames):
        return {'pixel': {'camera0': frames.view(self.N, *self.frame_shape)}}

    def _result(self):
        return self._obs(self.state), self.reward, self.done, {'obs_next': self._obs(self.obs_next)}

    def observation_spec(self):
        return {'pixel': {'camera0': self.frame_shape}}

    def reset(self):
        self.state.copy_(torch.randint(0, 256, (self.N, self.frame_bytes), generator=self._g, dtype=torch.uint8).to(self.device))
        self.ep_step.zero_()
        return self._obs(self.state), {}

"""Experience-sender wrappers for BATCHED envs, device-resident or on the host (mirror of
surreal/env/exp_sender_wrapper.py:72-112,153-264).

The reference keeps one Python deque per actor process and ships finished windows / n-step transitions
through pyarrow + ZeroMQ to the replay server.  Here the N deques are HBM arrays, the "send" is a kernel
that copies the record into the HBM replay's ring in (step, actor) order, and the md5 de-duplication of
overlapping windows (exp_sender.py:10-59) has nothing left to do."""
import ctypes as C

import torch

from .. import _lib
from .._lib import check
from ..distributed import LocalHub
from ..session import ConfigError
from ..utils import obs_flat, obs_source, record_action_dim


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _st():
    from ..ops import _stream
    return _stream()


class _WrapperBase:
    def __init__(self, env, learner_config, session_config, replay=None, obs_extra=0):
        self.env = env
        self.learner_config = learner_config
        self.session_config = session_config
        self.replay = replay if replay is not None else LocalHub.get(session_config).replays.get(0)
        if self.replay is None:
            raise RuntimeError('no replay registered for this session: construct the Replay before the agent '
                               'wraps its env (the ZeroMQ collector address of the reference is gone)')
        # D: floats per staged observation row = the env's obs_dim + obs_extra trailing floats (an RNN agent's LSTM cells,
        # utils.record_obs_dim)
        # A: floats per staged action = the replay's record width (utils.record_action_dim: 1 for a discrete spec)
        self.N, self.D = env.N, env.D + int(obs_extra)
        self.A = record_action_dim(self.replay.env_config.action_spec)
        self.obs_dim = env.D
        # a batched HOST env (numpy in / numpy out, attributes N, D, A) has no device: the staging lives with the replay
        self.device = env.device if hasattr(env, 'device') else self.replay.device
        self.host_env = not hasattr(env, 'device')
        self._pins, self._devs = {}, {}
        self._last_obs_host, self._last_obs_dev = None, None
        if not hasattr(env, 'step_counter'):
            self.step_counter = torch.zeros(1, dtype=torch.int64, device=self.device)   # Philox step counter

    def _h2d(self, name, arr, shape):
        """numpy -> device through a persistent pinned staging buffer (skipped when ``arr`` already is pinned)."""
        import numpy as np
        dev = self._devs.get(name)
        if dev is None:
            dev = self._devs[name] = torch.zeros(*shape, dtype=torch.float32, device=self.device)
        src = None
        if isinstance(arr, np.ndarray) and arr.dtype == np.float32 and arr.flags['C_CONTIGUOUS'] and arr.flags['WRITEABLE']:
            t = torch.from_numpy(arr)
            if t.is_pinned():
                src = t.view(*shape)
        if src is None:
            pin = self._pins.get(name)
            if pin is None:
                pin = self._pins[name] = torch.empty(*shape, dtype=torch.float32, pin_memory=True)
            pin.numpy()[...] = np.asarray(arr, dtype=np.float32).reshape(shape)
            src = pin
        dev.copy_(src, non_blocking=True)
        return dev

    def _dev(self, name, shape, dtype=torch.float32):
        dev = self._devs.get(name)
        if dev is None:
            dev = self._devs[name] = torch.zeros(*shape, dtype=dtype, device=self.device)
        return dev

    def _pinned(self, name, arr, shape, dtype=torch.float32):
        """Address (c_void_p) of ``arr`` if it already lives in pinned memory, else of a pinned staging copy."""
        import numpy as np
        npt = np.float64 if dtype == torch.float64 else np.float32
        if isinstance(arr, np.ndarray) and arr.dtype == npt and arr.flags['C_CONTIGUOUS'] and arr.flags['WRITEABLE'] \
                and torch.from_numpy(arr).is_pinned():
            return C.c_void_p(arr.ctypes.data)
        pin = self._pins.get(name)
        if pin is None:
            pin = self._pins[name] = torch.empty(*shape, dtype=dtype, pin_memory=True)
        pin.numpy()[...] = np.asarray(arr, dtype=npt).reshape(shape)
        return C.c_void_p(pin.data_ptr())

    def cached_device_obs(self, obs_arr):
        """The device copy of the observation the last step() returned (the agent's next act() input), if
        ``obs_arr`` is that very array: saves the second H2D of the same 256 KB."""
        return self._last_obs_dev if (obs_arr is not None and obs_arr is self._last_obs_host) else None

    @property
    def unwrapped(self):
        return getattr(self.env, 'unwrapped', self.env)

    def __getattr__(self, k):
        return getattr(self.env, k)


class ExpSenderWrapperMultiStepMovingWindowWithInfo(_WrapperBase):
    """n_step windows with stride (exp_sender_wrapper.py:153-264) -> FIFOReplay ring."""

    def __init__(self, env, learner_config, session_config, replay=None, cells=None):
        # RNN policy: the agent's (h, c) cells [layers, N, H], which every staged observation row carries behind the env's
        # observation (utils.rnn_cell_layout), as they are when the row is staged
        self.cells = cells
        extra = 0 if cells is None else 2 * cells[0].shape[0] * cells[0].shape[2]
        super().__init__(env, learner_config, session_config, replay, obs_extra=extra)
        self.n_step = self.learner_config.algo.n_step
        self.stride = self.learner_config.algo.stride
        if self.stride < 1:
            raise ConfigError('stride {} for experience generation cannot be less than 1'.format(self.stride))
        N, n, D, A = self.N, self.n_step, self.D, self.A
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        self.stage_pos = torch.zeros(N, dtype=torch.int32, device=self.device)
        self.stage_obs, self.stage_act, self.stage_pd = f(N, n + 1, D), f(N, n, A), f(N, n, 2 * A)
        self.stage_rew, self.stage_done = f(N, n), f(N, n)
        self._dest = torch.zeros(N, dtype=torch.int32, device=self.device)
        self._slots_ready = False      # the agent's sampling kernel already assigned this step's replay slots
        self.fuse_launches = True      # sample+assign / env+commit: 3 launches per step instead of 5 (same results)
        self.persistent_rollout = True  # device env + supported policy: whole chunks in ONE launch (agent.rollout_chunk)
        self.wide_commit = False       # RNN records: commit without shared-memory staging at any row width (same bytes)
        self._outbox = {}
        r = self.replay
        assert (r.n_step, r.D, r.A) == (n, D, A), 'replay record shape does not match the env / n_step'
        # every buffer the staging entries take, by name: allocated above and in the replay, never reallocated
        ptrs = {k: getattr(self, k).data_ptr() for k in ('stage_pos', 'stage_obs', 'stage_act', 'stage_pd', 'stage_rew',
                                                         'stage_done', 'step_counter')}
        ptrs.update({k: getattr(r, k).data_ptr() for k in ('r_obs', 'r_act', 'r_pd', 'r_rew', 'r_done')})
        self.windows = _lib.Windows(N=N, n_step=n, stride=self.stride, D=D, A=A, dest=self._dest.data_ptr(),
                                    fifo_state=r.state.data_ptr(), **ptrs)
        # the step's rows: the cells are fixed, the rows themselves are filled per step
        self._rows = _lib.WindowRows(obs_dim=self.obs_dim)
        if cells is not None:
            h, c = cells
            self._rows.layers, self._rows.H, self._rows.h, self._rows.c = h.shape[0], h.shape[2], h.data_ptr(), c.data_ptr()

    def reset(self):
        obs, info = self.env.reset()
        self.stage_pos.zero_()                                     # deque.clear() (exp_sender_wrapper.py:204-207)
        o = obs_flat(obs)
        row0 = self.stage_obs[:, 0]
        if self.host_env:
            d = self._h2d('obs', o, (self.N, self.obs_dim))
            row0[:, :self.obs_dim].copy_(d)
            self._last_obs_host, self._last_obs_dev = obs_source(obs), d
        else:
            row0[:, :self.obs_dim].copy_(o)
        if self.cells is not None:                                 # the cells the agent acts from on this observation
            h, c = self.cells
            L, H = h.shape[0], h.shape[2]
            row0[:, self.obs_dim:self.obs_dim + L * H].unflatten(1, (L, H)).copy_(h.transpose(0, 1))
            row0[:, self.obs_dim + L * H:].unflatten(1, (L, H)).copy_(c.transpose(0, 1))
        return obs, info

    def rollout_outbox(self, T):
        """Buffers of the persistent rollout kernel for chunks of T steps: per-actor outbox of finished windows (in
        the replay's record layout), their completion steps, and the commit pass's scratch.  None when the outbox
        would not be worth its memory (tiny strides)."""
        key = int(T)
        if key in self._outbox:
            return self._outbox[key]
        N, n, D, A = self.N, self.n_step, self.D, self.A
        W = T // self.stride + 2
        rec_bytes = 4 * ((n + 1) * D + n * A + n * 2 * A + 2 * n)
        ob = None
        if N * W * rec_bytes <= 4 << 30:
            f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
            z = lambda k: torch.zeros(k, dtype=torch.int32, device=self.device)      # noqa: E731
            ob = dict(W=W, o_obs=f(N * W, n + 1, D), o_act=f(N * W, n, A), o_pd=f(N * W, n, 2 * A), o_rew=f(N * W, n),
                      o_done=f(N * W, n), ev_step=z(N * W), ev_count=z(N),
                      scratch=z(int(_lib.lib().sb200_ppo_rollout_scratch_ints(N, W, T))))
        self._outbox[key] = ob
        return ob

    def mark_slots_assigned(self):
        """PPOAgent.act folds this step's slot assignment into its sampling launch (sb200_ppo_sample_f32 with
        assign_slots): the following step() then skips its own assignment pass."""
        self._slots_ready = True

    def step(self, action):
        """``action`` = (action_choice, action_info) as PPOAgent.act returns in training mode; the agent has
        already staged action / pd rows for this step (sb200_ppo_sample_f32).  An RNN policy's rows get the cells the
        agent holds NOW, i.e. the ones it acts from on the next observation (`on` and `o` differ only where an episode
        ended)."""
        a = action[0] if isinstance(action, tuple) else action
        ready, self._slots_ready = self._slots_ready, False
        if ready and hasattr(self.env, 'step_and_commit_window') and self.cells is None:
            return self.env.step_and_commit_window(a, self)        # env step + commit in ONE launch
        obs, reward, done, info = self.env.step(a)
        o = obs_flat(obs)
        on = obs_flat(info['obs_next']) if (isinstance(info, dict) and 'obs_next' in info) else o
        rows, N, Do = self._rows, self.N, self.obs_dim
        if self.host_env:
            # host env: this step's successor observation / reward / done cross PCIe (uint8 frames as their 32-bit words),
            # issued with the staging kernels from ONE C call; the device copy of the next observation is handed to the
            # agent's next act() (cached_device_obs, keyed by the array the env returned)
            rows.obs_reset_host = self._pinned('obs', o, (N, Do))
            rows.obs_next_host = rows.obs_reset_host if on is o else self._pinned('obs_next', on, (N, Do))
            rows.reward_host, rows.done_host = self._pinned('rew', reward, (N,)), self._pinned('done', done, (N,))
            d_o = self._dev('obs', (N, Do))
            rows.obs_reset, rows.obs_next = d_o.data_ptr(), self._dev('obs_next', (N, Do)).data_ptr()
            rows.reward, rows.done = self._dev('rew', (N,)).data_ptr(), self._dev('done', (N,)).data_ptr()
        else:
            rows.obs_next, rows.obs_reset, rows.reward, rows.done = on.data_ptr(), o.data_ptr(), reward.data_ptr(), done.data_ptr()
        rows.slots_assigned, rows.force_wide = int(ready), int(self.wide_commit)
        check(_lib.lib().sb200_ppo_window_step_f32(C.byref(self.windows), C.byref(rows), _st()), 'sb200_ppo_window_step_f32')
        if self.host_env:
            self._last_obs_host, self._last_obs_dev = obs_source(obs), d_o
        return obs, reward, done, info


class ExpSenderWrapperSSARNStepBootstrap(_WrapperBase):
    """n-step bootstrapped SSAR transitions (exp_sender_wrapper.py:72-112) -> UniformReplay ring."""

    def __init__(self, env, learner_config, session_config, replay=None):
        super().__init__(env, learner_config, session_config, replay)
        self.n_step = self.learner_config.algo.n_step
        self.gamma = self.learner_config.algo.gamma
        N, n, D, A = self.N, self.n_step, self.D, self.A
        self.dq_len = torch.zeros(N, dtype=torch.int32, device=self.device)
        self.dq_obs = torch.zeros(N, n, D, device=self.device)
        self.dq_act = torch.zeros(N, n, A, device=self.device)
        self.dq_rew = torch.zeros(N, n, dtype=torch.float64, device=self.device)
        self._dest = torch.zeros(N, dtype=torch.int32, device=self.device)
        self._emit = torch.zeros(N, device=self.device)
        self._obs = torch.zeros(N, D, device=self.device)
        # every buffer the staging entries take, by name: allocated above and in the replay, never reallocated
        r = self.replay
        ptrs = {k: getattr(self, k).data_ptr() for k in ('dq_len', 'dq_obs', 'dq_act', 'dq_rew', 'step_counter')}
        ptrs.update({k: getattr(r, k).data_ptr() for k in ('r_obs', 'r_obs_next', 'r_act', 'r_rew', 'r_done')})
        self.ssar = _lib.Ssar(N=N, n_step=n, gamma=float(self.gamma), D=D, A=A, dest=self._dest.data_ptr(),
                              emit=self._emit.data_ptr(), uniform_state=r.state.data_ptr(), **ptrs)

    def reset(self):
        obs, info = self.env.reset()
        self.dq_len.zero_()
        if self.host_env:
            import numpy as np
            o = obs_flat(obs)
            self._obs.copy_(torch.from_numpy(np.ascontiguousarray(o, dtype=np.float32)).view(self.N, self.D))
            self._last_obs_host, self._last_obs_dev = o, self._obs
        else:
            self._obs.copy_(obs['low_dim']['flat_inputs'])
        return obs, info

    def step(self, action):
        """``action``: what the env steps with, or the pair (env action, record action) of a discrete agent (QAgent.act:
        one-hot rows for the env, the indices as floats for the record)."""
        obs, reward, done, info = self.env.step(action)
        if isinstance(action, tuple):
            action = action[1]
        if self.host_env:
            self._step_host(obs, action, reward, done, info)
            return obs, reward, done, info
        check(_lib.lib().sb200_ssar_step_f32(C.byref(self.ssar), _p(self._obs), _p(action), _p(info['obs_next']), _p(reward),
                                             _p(done), _st()), 'sb200_ssar_step_f32')
        self.replay.mark_device_inserts()
        self._obs.copy_(obs['low_dim']['flat_inputs'])             # s_t of the next transition (reset obs where done)
        return obs, reward, done, info

    def _step_host(self, obs, action, reward, done, info):
        """A host env's step in ONE C call (sb200_ssar_step_host_f32): successor, action, done and the float64 rewards
        cross PCIe, the n-step sums stay float64 until emission, and s_t of the next transition is left in ``_obs`` --
        the device copy the agent's next act() reuses (cached_device_obs)."""
        N, D, A = self.N, self.D, self.A
        o = obs_flat(obs)
        on = info['obs_next'] if (isinstance(info, dict) and 'obs_next' in info) else o
        h_o = self._pinned('obs', o, (N, D))
        h_on = h_o if on is o else self._pinned('obs_next', on, (N, D))
        check(_lib.lib().sb200_ssar_step_host_f32(
            C.byref(self.ssar), h_on, h_o, self._pinned('act', action, (N, A)), self._pinned('rew', reward, (N,), torch.float64),
            self._pinned('done', done, (N,)), _p(self._obs), _p(self._dev('obs_next', (N, D))), _p(self._dev('act', (N, A))),
            _p(self._dev('rew', (N,), torch.float64)), _p(self._dev('done', (N,))), _st()), 'sb200_ssar_step_host_f32')
        self.replay.mark_device_inserts()
        self._last_obs_host, self._last_obs_dev = o, self._obs

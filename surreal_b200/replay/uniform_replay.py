"""UniformReplay in HBM (drop-in for surreal/replay/uniform_replay.py:6-74).

Storage: SoA ring of ``memory_size`` SSAR records -- obs [C][D], obs_next [C][D], act [C][A], rew [C],
done [C] (552 B per record at D=64, A=8; 1 M records = 552 MB of the 180 GB HBM3e).  The k-th insert lands
in slot k % memory_size, on-device actors insert through the ssar_step kernel (no host round trip).

Sampling is bit-exact with the reference: ``batch_size`` i.i.d. ``random.randint(0, len-1)`` draws WITH
replacement.  The draws come from a C++ MT19937 that continues Python's *global* ``random`` stream (state
transplanted in, advanced state written back), 16 KB of indices are uploaded, and a gather kernel assembles
the batch (aggregator.py:52-103 layout: rewards / dones as [B,1]).

``sample_device`` is the second sampler: Philox indices drawn ON the device over a sampling view that also lives there,
and the gather, in one launch (sb200_uniform_sample_gather_f32).  It never touches the host, so it can sit inside a CUDA
graph next to the learner's update; its index stream is its own (not ``random.randint``'s), which is why ``sample``
stays the default and the parity path."""
import ctypes as C
import random

import numpy as np
import torch

from .. import _lib
from .._lib import check
from ..ops import _ptr, _stream
from ..staging import Staging
from ..utils import record_action_dim
from .base import Replay, gather_fields


class PyRandomStream:
    """Index stream identical to ``rng.randint(0, m-1)`` of a Python ``random.Random`` (default: the
    module-level generator the reference uses), produced in C++ and kept in lock-step with it."""

    def __init__(self, rng=None):
        self.rng = rng
        L = _lib.lib()
        self._state = (C.c_uint8 * L.sb200_mt19937_state_bytes())()
        self._words = (C.c_uint32 * 624)()
        self._index = C.c_int(0)

    def randint_fill(self, population, count, out_np):
        L = _lib.lib()
        src = self.rng if self.rng is not None else random
        ver, internal, gauss = src.getstate()
        for i in range(624):
            self._words[i] = internal[i]
        check(L.sb200_mt19937_set_state_h(self._state, self._words, int(internal[624])), 'mt19937_set_state')
        check(L.sb200_mt19937_randint_fill_h(self._state, int(population), int(count),
                                             out_np.ctypes.data_as(C.c_void_p)), 'mt19937_randint_fill')
        check(L.sb200_mt19937_get_state_h(self._state, self._words, C.byref(self._index)), 'mt19937_get_state')
        src.setstate((ver, tuple(self._words) + (self._index.value,), gauss))


class UniformReplay(Replay):
    def __init__(self, learner_config, env_config, session_config, index=0):
        super().__init__(learner_config, env_config, session_config, index)
        if not torch.cuda.is_available():
            raise RuntimeError('surreal_b200.UniformReplay lives in HBM: a CUDA device is required')
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.memory_size = self.learner_config.replay.memory_size
        self.batch_size = self.learner_config.replay.batch_size
        self.D = sum(v[0] for v in self.env_config.obs_spec['low_dim'].values())
        self.A = record_action_dim(self.env_config.action_spec)
        C_, D, A = self.memory_size, self.D, self.A
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        self.r_obs, self.r_obs_next, self.r_act = f(C_, D), f(C_, D), f(C_, A)
        self.r_rew, self.r_done = f(C_), f(C_)
        assert _lib.lib().sb200_uniform_state_bytes() == 32
        self.state = torch.zeros(4, dtype=torch.int64, device=self.device)    # next_idx, size, capacity, total_in
        self.state[2] = C_
        self._host_size = 0               # mirror of `size`; refreshed from the device when actors insert there
        self._host_next = 0
        self._dirty = False
        self.stream = PyRandomStream()
        self._staging = Staging(self.device)    # host inserts: the record; sample: the indices
        self._idx_event = None
        # device sampler: the view {start, count, capacity} it draws from, its {draw counter, status} block and the seed
        rc = self.learner_config.replay
        self.sampler_seed = int(rc.sampler_seed) if 'sampler_seed' in rc else 0
        assert _lib.lib().sb200_uniform_sampler_bytes() == 16
        self.view = torch.zeros(3, dtype=torch.int64, device=self.device)
        self.sampler = torch.zeros(2, dtype=torch.int64, device=self.device)
        self._dev_indices = torch.zeros(self.batch_size, dtype=torch.int64, device=self.device)

    def mark_device_inserts(self):
        """Called by the on-device experience wrapper: the control block changed on the GPU."""
        self._dirty = True

    def _sync_state(self):
        if self._dirty:
            s = self.state.cpu().numpy()
            self._host_next, self._host_size = int(s[0]), int(s[1])
            self._dirty = False

    def __len__(self):
        self._sync_state()
        return self._host_size

    def start_sample_condition(self):
        return len(self) > self.learner_config.replay.sampling_start_size     # strict (uniform_replay.py:70-71)

    def evict(self):
        raise NotImplementedError

    def insert(self, exp):
        """Host insert of one SSAR dict {obs: [s, s'], action, reward, done} (exp_sender_wrapper.py:54-70)."""
        self._sync_state()
        D, A = self.D, self.A
        flat = lambda o: np.concatenate([np.asarray(o['low_dim'][k], dtype=np.float32).reshape(-1)  # noqa: E731
                                         for k in o['low_dim']])
        pin = self._staging.pinned('record', (2 * D + A + 2,))
        buf = pin.numpy()
        buf[:D], buf[D:2 * D] = flat(exp['obs'][0]), flat(exp['obs'][1])
        buf[2 * D:2 * D + A] = np.asarray(exp['action'], dtype=np.float32)
        buf[2 * D + A], buf[2 * D + A + 1] = np.float32(exp['reward']), np.float32(exp['done'])
        stage = self._staging.device('record', pin.shape)
        stage.copy_(pin)                                          # synchronous: the next insert rewrites the pinned record
        slot = self._host_next
        self.r_obs[slot].copy_(stage[:D])
        self.r_obs_next[slot].copy_(stage[D:2 * D])
        self.r_act[slot].copy_(stage[2 * D:2 * D + A])
        self.r_rew[slot] = stage[2 * D + A]
        self.r_done[slot] = stage[2 * D + A + 1]
        self._host_next = (slot + 1) % self.memory_size
        self._host_size = min(self._host_size + 1, self.memory_size)
        self.state[0], self.state[1] = self._host_next, self._host_size
        self.state[3] += 1

    def sample_indices(self, batch_size):
        """-> int64 numpy array: exactly [random.randint(0, len-1) for _ in range(batch_size)]."""
        n = len(self)
        if self._idx_event is not None:
            self._idx_event.synchronize()                         # the previous batch's H2D copy has consumed the buffer
        out = self._staging.pinned('indices', (batch_size,), np.int64).numpy()
        self.stream.randint_fill(n, batch_size, out)
        return out

    def sample(self, batch_size, out=None):
        L = _lib.lib()
        D, A = self.D, self.A
        self.sample_indices(batch_size)
        st = self._staging
        pin, idx = st.pinned('indices', (batch_size,), np.int64), st.device('indices', (batch_size,), np.int64)
        st.upload('indices', pin, idx)
        if self._idx_event is None:
            self._idx_event = torch.cuda.Event()
        self._idx_event.record()                                  # refilling the pinned buffer waits for this copy
        indices = pin.clone()                                     # the caller's copy: later samples do not alias it
        if out is None:
            f = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)  # noqa: E731
            out = dict(obs=f(batch_size, D), obs_next=f(batch_size, D), actions=f(batch_size, A),
                       rewards=f(batch_size, 1), dones=f(batch_size, 1))
        gather_fields([(self.r_obs, out['obs'], D), (self.r_obs_next, out['obs_next'], D), (self.r_act, out['actions'], A),
                       (self.r_rew, out['rewards'], 1), (self.r_done, out['dones'], 1)], None, idx, batch_size)
        return {'obs': {'low_dim': {'flat_inputs': out['obs']}}, 'obs_next': {'low_dim': {'flat_inputs': out['obs_next']}},
                'actions': out['actions'], 'rewards': out['rewards'], 'dones': out['dones'],
                'indices': indices}

    # -- device sampler ----------------------------------------------------------------------------------
    def snapshot_view(self, reserve=0):
        """Fix the population ``sample_device`` draws from: every record in the ring now, minus the slots the next
        ``reserve`` inserts can overwrite (sb200_uniform_view).  One one-thread launch on the current stream; call it
        where that stream is ordered after the inserts so far and before the next ones."""
        check(_lib.lib().sb200_uniform_view(_ptr(self.state), int(reserve), _ptr(self.view), _stream()), 'sb200_uniform_view')

    @property
    def draw_counter(self):
        """Sample launches that have drawn so far (host read: synchronises)."""
        return int(self.sampler[0])

    @property
    def sampler_status(self):
        """1 when the last ``sample_device`` found an empty view and sampled nothing (host read: synchronises)."""
        return int(self.sampler.view(torch.int32)[2])

    def sample_device(self, batch_size, out=None):
        """The batch dict of ``sample`` drawn from ``self.view`` without the host: no fill-level read, no pinned buffer,
        no event -- one launch, capturable.  ``indices`` is a device tensor owned by the replay (overwritten by the next
        call); a batch size other than ``replay.batch_size`` must be used once outside a capture first."""
        D, A = self.D, self.A
        if self._dev_indices.numel() < batch_size:
            self._dev_indices = torch.zeros(batch_size, dtype=torch.int64, device=self.device)
        idx = self._dev_indices[:batch_size]
        if out is None:
            f = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)  # noqa: E731
            out = dict(obs=f(batch_size, D), obs_next=f(batch_size, D), actions=f(batch_size, A),
                       rewards=f(batch_size, 1), dones=f(batch_size, 1))
        pairs = [(self.r_obs, out['obs'], D), (self.r_obs_next, out['obs_next'], D), (self.r_act, out['actions'], A),
                 (self.r_rew, out['rewards'], 1), (self.r_done, out['dones'], 1)]
        n = len(pairs)
        srcs = (C.c_void_p * n)(*[p[0].data_ptr() for p in pairs])
        outs = (C.c_void_p * n)(*[p[1].data_ptr() for p in pairs])
        recs = (C.c_int64 * n)(*[int(p[2]) for p in pairs])
        check(_lib.lib().sb200_uniform_sample_gather_f32(srcs, outs, recs, n, _ptr(self.view), self.sampler_seed,
                                                         _ptr(self.sampler), int(batch_size), _ptr(idx), _stream()),
              'sb200_uniform_sample_gather_f32')
        return {'obs': {'low_dim': {'flat_inputs': out['obs']}}, 'obs_next': {'low_dim': {'flat_inputs': out['obs_next']}},
                'actions': out['actions'], 'rewards': out['rewards'], 'dones': out['dones'], 'indices': idx}

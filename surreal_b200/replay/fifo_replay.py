"""FIFOReplay in HBM (drop-in for surreal/replay/fifo_replay.py:6-48).

Storage is a ring of ``memory_size + 3`` window records (SoA, record-major):
  obs  [C][n+1][D]  (row n is obs_next)   act [C][n][A]   pd [C][n][2A]   rew [C][n]   done [C][n]
with the queue control block {head, count, capacity, dropped, total_in, total_out} ALSO in device memory,
so on-device actors push windows without any host round trip.  Semantics are the reference's exactly:
arrival order out, silent drop of the OLDEST at capacity, ready when len >= batch_size.

``sample()`` pops the oldest ``batch_size`` windows and gathers them into the learner-facing batch
(the aggregator's layout, aggregator.py:176-183) as CUDA tensors."""
import numpy as np
import torch

from .. import _lib
from .._lib import check
from ..ops import _ptr, _stream
from ..staging import Staging
from ..utils import pack_window_records
from .base import Replay, gather_fields


class FIFOReplay(Replay):
    def __init__(self, learner_config, env_config, session_config, index=0):
        super().__init__(learner_config, env_config, session_config, index)
        self.batch_size = self.learner_config.replay.batch_size
        self.memory_size = self.learner_config.replay.memory_size
        assert self.session_config.replay.max_puller_queue <= 10
        assert self.session_config.replay.max_prefetch_queue == 1
        assert not self.session_config.sender.flush_time
        assert self.session_config.sender.flush_iteration <= 10
        if not torch.cuda.is_available():
            raise RuntimeError('surreal_b200.FIFOReplay lives in HBM: a CUDA device is required')
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.n_step = self.learner_config.algo.n_step
        from ..utils import record_obs_dim, obs_packed_dim, obs_is_pixel, rnn_cell_layout
        self.D = record_obs_dim(self.learner_config, self.env_config)   # pixel frames: opaque 32-bit words; RNN: + LSTM cells
        self.cells = rnn_cell_layout(self.learner_config, self.env_config)
        self.obs_dim = obs_packed_dim(self.env_config.obs_spec)
        self.pixel_shape = tuple(self.env_config.obs_spec['pixel']['camera0']) if obs_is_pixel(self.env_config.obs_spec) else None
        self.A = self.env_config.action_spec.dim[0]
        self.capacity = self.memory_size + 3                    # "+ 3 for a gentle buffering" (fifo_replay.py:27)
        C_, n, D, A = self.capacity, self.n_step, self.D, self.A
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        self.r_obs, self.r_act, self.r_pd = f(C_, n + 1, D), f(C_, n, A), f(C_, n, 2 * A)
        self.r_rew, self.r_done = f(C_, n), f(C_, n)
        L = _lib.lib()
        nb = int(L.sb200_fifo_state_bytes())                    # {head, count, capacity, dropped, int64 in, out, ...}
        assert nb >= 32 and nb % 4 == 0
        self.state = torch.zeros(nb // 4, dtype=torch.int32, device=self.device)
        self.state[2] = self.capacity
        self._idx = torch.zeros(max(self.batch_size, 1), dtype=torch.int32, device=self.device)
        self._status = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._slots = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._staging = Staging(self.device)                    # host inserts: the record, pinned and on the device
        self.check_underflow = True

    # -- control block ---------------------------------------------------------------------------------
    def _read_state(self):
        s = self.state.cpu().numpy()
        return dict(head=int(s[0]), count=int(s[1]), capacity=int(s[2]), dropped=int(s[3]),
                    total_in=int(s[4:6].view(np.int64)[0]), total_out=int(s[6:8].view(np.int64)[0]))

    def __len__(self):
        return self._read_state()['count']

    def start_sample_condition(self):
        return len(self) >= self.batch_size

    def evict(self):
        raise NotImplementedError('no support for eviction in FIFO mode')

    # -- host insert (external / CPU actors) -----------------------------------------------------------
    def insert(self, exp):
        """``exp``: the dict ExpSenderWrapperMultiStepMovingWindowWithInfo.send emits
        (exp_sender_wrapper.py:244-264): obs [n dicts], obs_next, actions, rewards, dones, persistent_infos."""
        n, D, A = self.n_step, self.D, self.A
        frames = self.pixel_shape is not None
        if frames:
            obs = lambda o: np.asarray(o['pixel']['camera0'], dtype=np.uint8)  # noqa: E731
        else:
            obs = lambda o: np.concatenate([np.asarray(o['low_dim'][k], dtype=np.float32).reshape(-1)  # noqa: E731
                                            for k in o['low_dim']])
        assert len(exp['obs']) == n, 'window length %d != n_step %d' % (len(exp['obs']), n)
        pin = self._staging.pinned('record', (n * (D + A + 2 * A + 2) + D,))
        buf = pin.numpy()
        o = (n + 1) * D
        # the cells [h, c], each [L, H], of the window's first step (ppo_agent.py:133-137); zeros when the window has none
        pack_window_records(buf[:o].reshape(1, n + 1, D), np.stack([obs(x) for x in exp['obs']]), obs(exp['obs_next']),
                            frames, self.cells, exp.get('onetime_infos') or None)
        buf[o:o + n * A] = np.stack(exp['actions']).astype(np.float32).reshape(-1); o += n * A
        buf[o:o + n * 2 * A] = np.stack([p[-1] for p in exp['persistent_infos']]).astype(np.float32).reshape(-1)
        o += n * 2 * A
        buf[o:o + n] = np.asarray(exp['rewards'], dtype=np.float32); o += n
        buf[o:o + n] = np.asarray(exp['dones'], dtype=np.float32)
        s = self._staging.device('record', pin.shape)
        self._staging.upload('record', pin, s)
        check(_lib.lib().sb200_fifo_push(_ptr(self.state), 1, _ptr(self._slots), _stream()), 'sb200_fifo_push')
        slot = int(self._slots.item())                          # host sync: the pinned record may be rewritten after it
        o = 0
        self.r_obs[slot].view(-1).copy_(s[o:o + (n + 1) * D]); o += (n + 1) * D
        self.r_act[slot].view(-1).copy_(s[o:o + n * A]); o += n * A
        self.r_pd[slot].view(-1).copy_(s[o:o + n * 2 * A]); o += n * 2 * A
        self.r_rew[slot].copy_(s[o:o + n]); o += n
        self.r_done[slot].copy_(s[o:o + n])

    # -- sample ------------------------------------------------------------------------------------------
    def sample(self, batch_size, out=None):
        """Pop the ``batch_size`` oldest windows (arrival order) -> aggregated device batch."""
        assert batch_size <= self.memory_size
        L = _lib.lib()
        n, D, A = self.n_step, self.D, self.A
        if self._idx.numel() < batch_size:
            self._idx = torch.zeros(batch_size, dtype=torch.int32, device=self.device)
        check(L.sb200_fifo_pop(_ptr(self.state), batch_size, _ptr(self._idx), _ptr(self._status), _stream()), 'sb200_fifo_pop')
        if out is None:
            f = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)  # noqa: E731
            out = dict(obs_full=f(batch_size, n + 1, D), actions=f(batch_size, n, A), pd=f(batch_size, n, 2 * A),
                       rewards=f(batch_size, n), dones=f(batch_size, n))
        gather_fields([(self.r_obs, out['obs_full'], (n + 1) * D), (self.r_act, out['actions'], n * A),
                       (self.r_pd, out['pd'], n * 2 * A), (self.r_rew, out['rewards'], n), (self.r_done, out['dones'], n)],
                      self._idx, None, batch_size)                      # all five fields: one launch
        if self.check_underflow and int(self._status.item()) != 0:      # host sync; the engine polls
            raise IndexError('pop from a FIFO replay holding fewer than %d windows' % batch_size)   # len() instead
        obs_full = out['obs_full']
        od = self.obs_dim
        onetime = None
        cl = self.cells
        if cl is not None:         # RNN policy: the LSTM cells of the window's first step ride behind the observation
            onetime = [cl.h(obs_full[:, 0]).unflatten(1, (cl.layers, cl.hidden)),
                       cl.c(obs_full[:, 0]).unflatten(1, (cl.layers, cl.hidden))]       # [B, L, H] views
        if self.pixel_shape is not None:
            fr = obs_full.view(torch.uint8).view(batch_size, n + 1, 4 * D)[:, :, :4 * od].unflatten(2, self.pixel_shape)
            return {'obs': {'pixel': {'camera0': fr[:, :n]}}, 'obs_next': {'pixel': {'camera0': fr[:, n:]}},
                    'obs_full': obs_full, 'actions': out['actions'], 'rewards': out['rewards'], 'dones': out['dones'],
                    'persistent_infos': [out['pd']], 'onetime_infos': onetime}
        return {'obs': {'low_dim': {'flat_inputs': obs_full[:, :n, :od]}},
                'obs_next': {'low_dim': {'flat_inputs': obs_full[:, n:, :od]}},
                'obs_full': obs_full, 'actions': out['actions'], 'rewards': out['rewards'], 'dones': out['dones'],
                'persistent_infos': [out['pd']], 'onetime_infos': onetime}

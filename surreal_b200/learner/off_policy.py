"""OffPolicyLearner: what DDPGLearner and DQNLearner share around their update (the algorithm, ``_optimize_device``).

A batch sits in fixed device buffers (``_own``, ``_w``) so that a captured CUDA graph always reads the same addresses.
``learn(batch)`` and ``learn_from_replay(replay, K)`` run one update body, K x [take the batch -> update -> priorities
back to a prioritized replay -> target update], as one graph per (replay, K, weighted), or the same launches eagerly
when graphs are off.  The kernels write the statistics, the latched stop flag and the target counter straight into one
device block, which the host reads back once per call."""
import numpy as np
import torch

from .. import _lib, ops
from .._lib import check
from ..ops import _ptr
from ..staging import Staging
from .base import Learner

_HEAD = 16                          # read-back block: int64 target counter [0:8], int32 stop flag [8:12], statistics [16:]


class OffPolicyLearner(Learner):
    """Subclasses build their networks and trainers, call ``_init_off_policy`` and provide ``_optimize_device(weights)``
    (one update on ``_own``), ``_target_pairs()`` ([(target net, online net)]), ``_statistics(stats, weighted)`` and
    ``bad_action_message``."""

    def _init_off_policy(self, obs_dim, action_width, n_stats, workspace, bad_offset, tau=None, counter=None, period=1,
                         incr=1):
        """``tau``: soft target updates; otherwise the hard copy counts ``incr`` per update in the host attribute named
        ``counter`` and copies when the count crosses a multiple of ``period``.  ``workspace[bad_offset:]`` holds the
        bad-action flag of the loss kernel."""
        B = self.batch_size
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        self._own = dict(obs=f(B, obs_dim), obs_next=f(B, obs_dim), actions=f(B, action_width), rewards=f(B, 1),
                         dones=f(B, 1))
        self._w = f(B, 1)                                      # learn(): the batch's importance weights
        self._prio = f(B)
        self._staging = Staging(self.device)              # numpy batches: pinned copies of ``_own``
        self._bad = workspace[bad_offset:bad_offset + 4].view(torch.int32)
        self._block = torch.zeros(_HEAD + 4 * n_stats, dtype=torch.uint8, device=self.device)
        self._counter = self._block[0:8].view(torch.int64)
        # latches the bad-action flag for the rest of the call: every later optimiser / priority / target kernel no-ops
        self._stop = self._block[8:12].view(torch.int32)
        self._stats_block = self._block[_HEAD:].view(torch.float32)
        self._tau, self._counter_attr, self._period, self._incr = tau, counter, int(period), int(incr)
        self.check_action_range = True
        self.use_cuda_graph = ops.graphs_enabled()
        self._graphs = {}

    # ------------------------------------------------------------------------------------------------
    def preprocess(self, batch):
        """Batch fields -> the fixed device buffers ``_own`` (numpy through pinned staging); device batches already in
        them are used in place."""
        get = (lambda k: batch[k]) if isinstance(batch, dict) else (lambda k: getattr(batch, k))
        flat = lambda o: o['low_dim']['flat_inputs'] if isinstance(o, dict) else o  # noqa: E731
        src = dict(obs=flat(get('obs')), obs_next=flat(get('obs_next')), actions=get('actions'),
                   rewards=get('rewards'), dones=get('dones'))
        self.last_h2d_bytes = sum(self._staging.upload(k, v, self._own[k]) for k, v in src.items())
        return batch

    def replay_out_buffers(self):
        return self._own

    @property
    def td_priorities(self):
        """Device [B]: the priorities of the last weighted update's rows (what a prioritized replay gets back)."""
        return self._prio

    def _latch_bad_action(self):
        """Raise the stop flag when the update's loss kernel flagged a bad action; returns the flag for the optimisers."""
        torch.maximum(self._stop, self._bad, out=self._stop)
        return self._stop

    def _update_targets(self):
        L, st = _lib.lib(), ops._stream()
        for i, (t, s) in enumerate(self._target_pairs()):
            if self._tau is not None:
                check(L.sb200_soft_update_f32(_ptr(t.params), _ptr(s.params), t.size, float(self._tau), _ptr(self._stop),
                                              st), 'sb200_soft_update_f32')
            else:
                check(L.sb200_hard_update_f32(_ptr(t.params), _ptr(s.params), t.size, _ptr(self._counter), self._period,
                                              self._incr, int(i == 0), _ptr(self._stop), st), 'sb200_hard_update_f32')

    def _updates_device(self, replay, K, weighted):
        """K x [batch -> update -> priorities (prioritized replay) -> target update] as one fixed launch sequence.  The
        batch comes from ``replay.sample_device`` or, without a replay, from what ``learn()`` put in ``_own``."""
        self._stop.zero_()
        for _ in range(K):
            if replay is None:
                self._optimize_device(self._w if weighted else None)
            else:
                b = replay.sample_device(self.batch_size, out=self._own)
                self._optimize_device(b['weights'] if weighted else None)
                if weighted:
                    replay.update_priorities_device(b['indices'], self._prio, stop_flag=self._stop)
            self._update_targets()

    def _run_updates(self, replay, K, weighted):
        if self._counter_attr is not None:
            self._counter.fill_(getattr(self, self._counter_attr))
        with self.forward_time.time():
            if self.use_cuda_graph:
                key = (None if replay is None else id(replay), K, weighted)
                if key not in self._graphs:
                    self._graphs[key] = (ops.GraphRunner(), replay)     # the replay is kept alive: its id stays unique
                self._graphs[key][0].run(lambda: self._updates_device(replay, K, weighted))
            else:
                self._updates_device(replay, K, weighted)

    def _finish(self, weighted):
        """The one read-back: target counter -> host attribute, the bad-action assert, statistics, logging."""
        rb = self._block.cpu().numpy()
        self.last_d2h_bytes = rb.nbytes
        if self._counter_attr is not None:
            setattr(self, self._counter_attr, int(rb[0:8].view(np.int64)[0]))
        if self.check_action_range and rb[8:12].view(np.int32)[0] != 0:
            raise AssertionError(self.bad_action_message)
        stats = self._statistics(rb[_HEAD:].view(np.float32), weighted)
        stats['performance/total_learn_time'] = self.total_learn_time.avg
        self.tensorplex.add_scalars(stats, global_step=self.current_iteration)
        self.periodic_checkpoint(global_steps=self.current_iteration, score=None)
        return stats

    def learn(self, batch):
        """One update on ``batch`` (ddpg.py:354-374, dqn.py:71-91).  A batch with ``weights`` (prioritized replay) takes
        the weighted loss; when it also carries ``indices`` and the attached replay has priorities, the new ones are
        written back to it.  An out-of-range action raises AssertionError after the update, which changed nothing."""
        self.current_iteration += 1
        get = (lambda k: batch.get(k)) if isinstance(batch, dict) else (lambda k: getattr(batch, k, None))
        weights, indices = get('weights'), get('indices')
        weighted = weights is not None
        with self.total_learn_time.time():
            self.preprocess(batch)
            if weighted:
                self._w.copy_(torch.as_tensor(weights, dtype=torch.float32).reshape(self._w.shape), non_blocking=True)
            self._run_updates(None, 1, weighted)
            if weighted and indices is not None and hasattr(self._replay, 'update_priorities_device'):
                idx = torch.as_tensor(indices, dtype=torch.int64).to(self.device).reshape(-1)
                self._replay.update_priorities_device(idx, self._prio, stop_flag=self._stop)
            return self._finish(weighted)

    def learn_from_replay(self, replay, updates=1):
        """``updates`` learner updates fed by ``replay.sample_device``, with no host step between them: one CUDA graph
        (the same launches eagerly when graphs are off), then ONE read-back.  Returns the statistics of the last update.
        The hard target counter lives on the device for the call: it starts from the host attribute and is read back
        into it.  An out-of-range action in any sampled batch raises AssertionError after the read-back; that update
        and every later one of the call changed nothing."""
        K = int(updates)
        assert K >= 1
        self.current_iteration += K
        weighted = hasattr(replay, 'update_priorities_device')
        with self.total_learn_time.time():
            self._run_updates(replay, K, weighted)
            return self._finish(weighted)

"""PrioritizedReplay in HBM: proportional prioritized experience replay (Schaul et al. 2016) over the UniformReplay ring,
following the reference's surreal/replay/prioritized_replay.py + segment_tree.py (openai-baselines form).

The ring, its control block, the SSAR insert paths and ``start_sample_condition`` are UniformReplay's.  On top of them
live a sum tree and a min tree of p^alpha over the ring's slots (fp32 leaves, fp64 internal sums), in device memory,
and three capturable entries (replay_per.cu):

  * ``snapshot_view``: admits every record inserted since the last admit at max_priority^alpha, then fixes the
    sampling view as UniformReplay does;
  * ``sample_device``: proportional draws over the view with their importance weights (leaf / min over view)^(-beta),
    and the gather of the drawn records, in one launch; beta follows the linear schedule of the reference's DQN on a
    device update counter, so the K updates of one graph each get their own beta;
  * ``update_priorities_device``: writes |td| + eps back as leaves p^alpha (the last of equal indices wins) and
    raises max_priority, unless the learner's stop flag is set.

Two bugs of the reference class (which cannot run as shipped) are fixed: a record's own slot gets its priority (the
reference writes the slot after it), and the mass is drawn over the whole view, newest record included (the reference
sums [0, len - 1))."""
import ctypes as C

import numpy as np
import torch

from .. import _lib
from .._lib import check
from ..ops import _ptr, _stream
from .uniform_replay import UniformReplay

# learner_config.replay keys read when present (the reference's PrioritizedReplay / DQN 'prioritized' defaults); a
# learner config with an algo.prioritized block (DQN) takes all four from there instead
PER_DEFAULTS = {'alpha': 0.6, 'beta0': 0.4, 'beta_anneal_iters': None, 'priority_eps': 1e-6}


class PrioritizedReplay(UniformReplay):
    def __init__(self, learner_config, env_config, session_config, index=0):
        super().__init__(learner_config, env_config, session_config, index)
        rc = self.learner_config.replay
        get = lambda k: rc[k] if k in rc else PER_DEFAULTS[k]  # noqa: E731
        algo = self.learner_config.algo
        if 'prioritized' in algo:                 # DQN's algo.prioritized block (dqn.py:115-119) is the one source there
            pc = algo.prioritized
            get = lambda k: pc['eps' if k == 'priority_eps' else k]  # noqa: E731
        self.alpha = float(get('alpha'))
        self.beta0 = float(get('beta0'))
        anneal = get('beta_anneal_iters')
        self.beta_anneal_iters = None if anneal is None else float(anneal)
        self.priority_eps = float(get('priority_eps'))
        if self.alpha < 0 or not 0 <= self.beta0 <= 1 or self.priority_eps <= 0:
            raise ValueError('prioritized replay needs alpha >= 0, 0 <= beta0 <= 1 and priority_eps > 0')
        L = _lib.lib()
        P, sub = C.c_int64(0), C.c_int64(0)
        check(L.sb200_per_tree_layout(self.memory_size, C.byref(P), C.byref(sub)), 'sb200_per_tree_layout')
        self.leaves, self.subtree = P.value, sub.value
        dev = self.device
        self.t_leaf = torch.zeros(P.value, dtype=torch.float32, device=dev)
        self.t_sum = torch.zeros(P.value, dtype=torch.float64, device=dev)
        self.t_min = torch.full((P.value,), float('inf'), dtype=torch.float32, device=dev)
        self.t_dirty = torch.zeros(P.value // sub.value, dtype=torch.int32, device=dev)
        self.t_owner = torch.full((self.memory_size,), -1, dtype=torch.int32, device=dev)
        assert L.sb200_per_ctrl_bytes() == 24
        self.ctrl = torch.zeros(3, dtype=torch.int64, device=dev)      # admitted, updates, {max_priority, ticket}
        self.ctrl.view(torch.float32)[4] = 1.0                          # max_priority starts at 1 (prioritized_replay.py:41)
        self.tree = _lib.PerTree(self.memory_size, P.value, sub.value, self.t_leaf.data_ptr(), self.t_sum.data_ptr(),
                                 self.t_min.data_ptr(), self.t_dirty.data_ptr(), self.t_owner.data_ptr(),
                                 self.ctrl.data_ptr())
        self._dev_weights = torch.zeros(self.batch_size, dtype=torch.float32, device=dev)
        self._full_view = torch.zeros(3, dtype=torch.int64, device=dev)
        self._host_upd = None

    # -- trees -------------------------------------------------------------------------------------------
    def admit(self):
        """Give every record inserted since the last admit max_priority^alpha, then rebuild the trees (device only)."""
        check(_lib.lib().sb200_per_admit(C.byref(self.tree), _ptr(self.state), self.alpha, _stream()), 'sb200_per_admit')

    def rebuild(self, full=False):
        """Recompute the internal nodes of the dirty subtrees (all of them with ``full``) and the levels above."""
        check(_lib.lib().sb200_per_rebuild(C.byref(self.tree), int(bool(full)), _stream()), 'sb200_per_rebuild')

    def priorities(self):
        """-> float32 numpy [memory_size]: the leaves p^alpha (0 for a slot never inserted).  Host read: synchronises."""
        return self.t_leaf[:self.memory_size].cpu().numpy()

    @property
    def max_priority(self):
        """Running max of every raw priority set, 1.0 at first (host read: synchronises)."""
        return float(self.ctrl.view(torch.float32)[4])

    @property
    def update_counter(self):
        """Sample launches that drew so far: the step t of the beta schedule (host read: synchronises)."""
        return int(self.ctrl[1])

    def beta(self, t):
        """LinearSchedule(beta_anneal_iters, beta0 -> 1) of the reference DQN (utils/schedule.py:96-99) at step t."""
        if self.beta_anneal_iters is None or self.beta_anneal_iters <= 0:
            return self.beta0
        return self.beta0 + min(float(t) / self.beta_anneal_iters, 1.0) * (1.0 - self.beta0)

    # -- sampling ----------------------------------------------------------------------------------------
    def snapshot_view(self, reserve=0):
        """Admit the records inserted so far, then fix the sampling view (UniformReplay.snapshot_view)."""
        self.admit()
        super().snapshot_view(reserve)

    def _sample(self, batch_size, out, view, beta_override):
        D, A = self.D, self.A
        if self._dev_indices.numel() < batch_size:
            self._dev_indices = torch.zeros(batch_size, dtype=torch.int64, device=self.device)
        if self._dev_weights.numel() < batch_size:
            self._dev_weights = torch.zeros(batch_size, dtype=torch.float32, device=self.device)
        idx, w = self._dev_indices[:batch_size], self._dev_weights[:batch_size]
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
        anneal = -1.0 if self.beta_anneal_iters is None else self.beta_anneal_iters
        check(_lib.lib().sb200_per_sample_gather_f32(C.byref(self.tree), srcs, outs, recs, n, _ptr(view), self.sampler_seed,
                                                     _ptr(self.sampler), int(batch_size), self.beta0, anneal,
                                                     float(beta_override), _ptr(idx), _ptr(w), _stream()),
              'sb200_per_sample_gather_f32')
        return {'obs': {'low_dim': {'flat_inputs': out['obs']}}, 'obs_next': {'low_dim': {'flat_inputs': out['obs_next']}},
                'actions': out['actions'], 'rewards': out['rewards'], 'dones': out['dones'], 'indices': idx,
                'weights': w.view(batch_size, 1)}

    def sample_device(self, batch_size, out=None):
        """UniformReplay.sample_device's batch drawn in proportion to the leaves over ``self.view``, plus ``weights``
        [B, 1], the importance weights at this update's beta.  ``indices`` and ``weights`` are device tensors owned by
        the replay (overwritten by the next call).  One launch, capturable."""
        return self._sample(batch_size, out, self.view, -1.0)

    def sample(self, batch_size, out=None, beta=None):
        """Host-driven sample (Learner.fetch_batch): admit, then draw with the device sampler over the whole filled
        ring.  ``beta`` overrides the schedule.  ``indices`` / ``weights`` are the caller's copies."""
        self.admit()
        n = len(self)
        self._full_view.copy_(torch.tensor([0, n, self.memory_size], dtype=torch.int64), non_blocking=False)
        b = self._sample(batch_size, out, self._full_view, -1.0 if beta is None else float(beta))
        b['indices'] = b['indices'].clone()
        b['weights'] = b['weights'].clone()
        return b

    # -- priorities --------------------------------------------------------------------------------------
    def update_priorities_device(self, indices, priorities, stop_flag=None):
        """leaf[indices[b]] = priorities[b]^alpha (the last of equal indices wins), max_priority = max(it, priorities),
        then the rebuild; a no-op while ``stop_flag`` (int32 device flag) is set.  Device tensors, capturable."""
        check(_lib.lib().sb200_per_update_f32(C.byref(self.tree), _ptr(indices), _ptr(priorities), int(indices.numel()),
                                              self.alpha, _ptr(stop_flag), _stream()), 'sb200_per_update_f32')

    def update_priorities(self, indices, priorities):
        """prioritized_replay.py:124-143 for host input (lists, numpy or CPU tensors), checked as the reference does
        (priority > 0, 0 <= index < len); device tensors go to ``update_priorities_device`` unchecked."""
        if isinstance(indices, torch.Tensor) and indices.is_cuda:
            return self.update_priorities_device(indices.to(torch.int64), priorities.reshape(-1).to(torch.float32))
        idx = np.asarray(indices, dtype=np.int64).reshape(-1)
        pr = np.asarray(priorities, dtype=np.float32).reshape(-1)
        assert len(idx) == len(pr)
        n = len(self)
        assert (pr > 0).all(), 'priorities must be positive'
        assert ((idx >= 0) & (idx < n)).all(), 'indices must lie in [0, len)'
        if len(idx) == 0:
            return None
        self._host_upd = (torch.from_numpy(idx).to(self.device), torch.from_numpy(pr).to(self.device))
        self.update_priorities_device(*self._host_upd)

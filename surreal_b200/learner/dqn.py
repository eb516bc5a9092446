"""DQNLearner: drop-in for surreal/learner/dqn.py:10-121 (low-dimensional observations) on hand-written kernels.

One update: the target towers (and, with double Q, the online towers) at s', the online towers at s with saved
activations, then ONE TD kernel (csrc/dqn.cu: dueling combine, argmax / gather, y = r + gamma (1 - done) q', Huber loss
weighted by the importance weights, the gradient rows of both towers, the priorities |td| + eps), the towers' backward
passes and one Adam step (eps 1e-4) over both towers with their gradient norm clipped jointly.  The target network is
copied whenever the running count of samples crosses a multiple of ``target_network_update_freq``
(PeriodicTracker.track_increment(batch_size), dqn.py:84-86)."""
import ctypes as C

import torch

from .. import _lib, ops
from .._lib import check
from .. import utils as U
from ..model.cnn_stem import joint_step
from ..model.q_net import QModel
from ..session import ConfigError
from .base import Learner

QS = dict(LOSS=0, TD_ERROR=1, Q=2, IS_WEIGHT=3, BAD_ROWS=4)
ADAM_EPS = 1e-4                                   # torch.optim.Adam(..., eps=1e-4), dqn.py:18-22


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def check_dqn_config(learner_config, env_config):
    """What DQN accepts: a discrete action spec, one-step records and no convolutional Q function."""
    spec = env_config.action_spec
    if not U.action_is_discrete(spec):
        raise ConfigError('DQN needs a discrete action spec, got %s' % (dict(spec),))
    if int(learner_config.algo.n_step) != 1:
        raise ConfigError('DQN bootstraps with gamma, not gamma^n (dqn.py:67): algo.n_step must be 1, got %s'
                          % learner_config.algo.n_step)
    if learner_config.model.convs:
        raise NotImplementedError('the convolutional Q function (q_net.py:68-119) is not built: model.convs must be empty')


def prioritized_eps(learner_config):
    """priority eps of the algo.prioritized block (dqn.py:115-119), the one source of the PER options."""
    return float(learner_config.algo.prioritized.eps)


class DQNLearner(Learner):
    def __init__(self, learner_config, env_config, session_config):
        super().__init__(learner_config, env_config, session_config)
        if not torch.cuda.is_available():
            raise RuntimeError('surreal_b200.DQNLearner needs a CUDA device (there is no CPU fallback)')
        check_dqn_config(self.learner_config, self.env_config)
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.current_iteration = 0
        lc = self.learner_config
        self.algo = lc.algo
        self.batch_size = B = int(lc.replay.batch_size)
        self.gamma = float(self.algo.gamma)
        self.double_q = bool(self.algo.double_q)
        self.n_actions = n = int(self.env_config.action_spec.dim[0])
        self.dueling = bool(lc.model.dueling)
        mk = dict(obs_spec=self.env_config.obs_spec, action_dim=n, fc_hidden_sizes=lc.model.fc_hidden_sizes,
                  dueling=self.dueling, convs=lc.model.convs, device=self.device)
        self.model = QModel(**mk)
        self.model_target = QModel(**mk)
        self.model_target.copy_from(self.model)                     # q_func.clone() (dqn.py:17)
        self.D = D = self.model.input_dim
        clip = self.algo.grad_norm_clipping
        self.optim_a = ops.MlpTrainer(self.model.action_net, B, self.algo.lr, clip_mode=0 if clip is None else 1,
                                      clip_value=0.0 if clip is None else float(clip), adam_eps=ADAM_EPS)
        self.optim_v = None
        if self.dueling:
            self.optim_v = ops.MlpTrainer(self.model.state_net, B, self.algo.lr, adam_eps=ADAM_EPS)
            self._grad = torch.zeros(self.model.action_net.size + self.model.state_net.size, dtype=torch.float32,
                                     device=self.device)
        self.target_update_period = int(self.algo.target_network_update_freq)
        self.target_update_samples = 0           # PeriodicTracker.value: samples consumed by updates so far
        self.priority_eps = prioritized_eps(lc)
        self.total_learn_time = U.TimeRecorder()
        self.forward_time = U.TimeRecorder()
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        Ar = U.record_action_dim(self.env_config.action_spec)
        self._own = dict(obs=f(B, D), obs_next=f(B, D), actions=f(B, Ar), rewards=f(B, 1), dones=f(B, 1))
        self._ta, self._tv = f(B, n), (f(B, 1) if self.dueling else None)             # target towers at s'
        self._oa, self._ov = f(B, n), (f(B, 1) if self.dueling else None)             # online towers at s' (double Q)
        self._stats = f(8)
        self._ws = torch.zeros(_lib.lib().sb200_dqn_workspace_bytes(B), dtype=torch.uint8, device=self.device)
        off = int(_lib.lib().sb200_dqn_bad_action_offset())
        self._bad = self._ws[off:off + 4].view(torch.int32)
        self._w = f(B, 1)
        self._prio = f(B)
        self.check_action_range = True
        self.use_cuda_graph = ops.graphs_enabled()
        self._graph, self._graph_w = ops.GraphRunner(), ops.GraphRunner()
        # learn_from_replay: one read-back buffer (float64: statistics [0:8], latched stop flag [8], sample counter [9])
        self._stop = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._samples = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._readback = torch.zeros(10, dtype=torch.float64, device=self.device)
        self._replay_graphs = {}

    # ------------------------------------------------------------------------------------------------
    def preprocess(self, batch):
        """Batch fields -> the learner's fixed device buffers (a captured graph always reads the same addresses)."""
        get = (lambda k: batch[k]) if isinstance(batch, dict) else (lambda k: getattr(batch, k))
        flat = lambda o: o['low_dim']['flat_inputs'] if isinstance(o, dict) else o  # noqa: E731
        src = dict(obs=flat(get('obs')), obs_next=flat(get('obs_next')), actions=get('actions'),
                   rewards=get('rewards'), dones=get('dones'))
        for k, v in src.items():
            dst = self._own[k]
            v = torch.as_tensor(v, dtype=torch.float32)
            if v.data_ptr() != dst.data_ptr():
                dst.copy_(v.reshape(dst.shape), non_blocking=True)
        return batch

    def replay_out_buffers(self):
        return self._own

    @property
    def td_priorities(self):
        """Device [B]: |td| + eps of the last weighted update's rows (the priorities to write back)."""
        return self._prio

    def _optimize_device(self, stop=None, weights=None):
        """dqn.py:44-69 + _run_optimizer as one fixed launch sequence (CUDA-graph body).  ``stop``: the flag that no-ops
        the optimiser -- this update's bad-action flag, or a flag that latches it.  ``weights`` (device [B, 1]): the
        importance weights of a prioritized batch; the rows' new priorities land in ``td_priorities``."""
        L, st = _lib.lib(), ops._stream()
        stop = self._bad if stop is None else stop
        b = self._own
        obs, obs_next = b['obs'], b['obs_next']
        self.model_target.forward_towers(obs_next, self._ta, self._tv)                   # q_target(s')
        if self.double_q:
            self.model.forward_towers(obs_next, self._oa, self._ov)                      # q_func(s') picks the column
        qa = self.optim_a.forward(obs)
        da = self.optim_a.d[-1]
        qv = dv = None
        if self.dueling:
            qv = self.optim_v.forward(obs)
            dv = self.optim_v.d[-1]
        oa, ov = (self._oa, self._ov) if self.double_q else (None, None)
        ld = lambda t: t.stride(0) if t is not None else 0  # noqa: E731
        check(L.sb200_dqn_td_f32(_ptr(qa), ld(qa), _ptr(qv), ld(qv), _ptr(self._ta), ld(self._ta), _ptr(self._tv),
                                 ld(self._tv), _ptr(oa), ld(oa), _ptr(ov), ld(ov), _ptr(b['actions']), _ptr(b['rewards']),
                                 _ptr(b['dones']), _ptr(weights), self.batch_size, self.n_actions, self.gamma,
                                 self.priority_eps, _ptr(da), ld(da), _ptr(dv), ld(dv),
                                 _ptr(self._prio if weights is not None else None), _ptr(self._stats), _ptr(self._ws),
                                 st), 'sb200_dqn_td_f32')
        if stop is not self._bad:
            torch.maximum(stop, self._bad, out=stop)
        self.optim_a.backward()
        if self.dueling:
            self.optim_v.backward()
            joint_step(self.optim_a, [self.optim_v], self._grad, stop_flag=stop, adam_eps=ADAM_EPS)
        else:
            self.optim_a.step(stop_flag=stop)

    def _statistics(self, s, weighted):
        stats = {'td_error': float(s[QS['TD_ERROR']]), 'loss': float(s[QS['LOSS']]), 'q_value': float(s[QS['Q']]),
                 'performance/forward_time': self.forward_time.avg}
        if weighted:
            stats['avg_is_weight'] = float(s[QS['IS_WEIGHT']])
        return stats

    def _target_crossed(self, samples_before):
        P = self.target_update_period
        return (samples_before + self.batch_size) // P > samples_before // P

    def learn(self, batch):
        """dqn.py:71-91.  A batch with ``weights`` (prioritized replay) takes the weighted loss; when it also carries
        ``indices`` and the attached replay has priorities, |td| + eps is written back to it (dqn.py:128-175)."""
        self.current_iteration += 1
        get = (lambda k: batch.get(k)) if isinstance(batch, dict) else (lambda k: getattr(batch, k, None))
        weights, indices = get('weights'), get('indices')
        with self.total_learn_time.time():
            self.preprocess(batch)
            if weights is not None:
                self._w.copy_(torch.as_tensor(weights, dtype=torch.float32).reshape(self._w.shape), non_blocking=True)
            with self.forward_time.time():
                if self.use_cuda_graph:
                    g = self._graph_w if weights is not None else self._graph
                    g.run(lambda: self._optimize_device(weights=self._w if weights is not None else None))
                else:
                    self._optimize_device(weights=self._w if weights is not None else None)
            if weights is not None and indices is not None and hasattr(self._replay, 'update_priorities_device'):
                idx = torch.as_tensor(indices, dtype=torch.int64).to(self.device).reshape(-1)
                self._replay.update_priorities_device(idx, self._prio, stop_flag=self._bad)
            s = self._stats.cpu().numpy()
            if self.check_action_range and s[QS['BAD_ROWS']] > 0:
                raise AssertionError('actions outside the integers [0, %d) (dqn.py:48)' % self.n_actions)
            if self._target_crossed(self.target_update_samples):                           # dqn.py:84-86
                self.model_target.copy_from(self.model)
            self.target_update_samples += self.batch_size
            stats = self._statistics(s, weights is not None)
            stats['performance/total_learn_time'] = self.total_learn_time.avg
            self.tensorplex.add_scalars(stats, global_step=self.current_iteration)
            self.periodic_checkpoint(global_steps=self.current_iteration, score=None)
        return stats

    def _replay_updates_device(self, replay, updates):
        """``updates`` x [sample on the device -> update -> priorities (PER) -> target gate] and the read-back staging, as
        one fixed launch sequence.  A bad-action batch stops every later optimiser / priority / target kernel (_stop)."""
        L, st = _lib.lib(), ops._stream()
        per = hasattr(replay, 'update_priorities_device')
        self._stop.zero_()
        for _ in range(updates):
            b = replay.sample_device(self.batch_size, out=self._own)
            self._optimize_device(stop=self._stop, weights=b['weights'] if per else None)
            if per:
                replay.update_priorities_device(b['indices'], self._prio, stop_flag=self._stop)
            for i, (t, s_) in enumerate(zip(self.model_target.nets(), self.model.nets())):
                check(L.sb200_hard_update_samples_f32(_ptr(t.params), _ptr(s_.params), t.size, _ptr(self._samples),
                                                      self.target_update_period, self.batch_size, int(i == 0),
                                                      _ptr(self._stop), st), 'sb200_hard_update_samples_f32')
        rb = self._readback
        rb[0:8].copy_(self._stats)
        rb[8:9].copy_(self._stop)
        rb[9:10].copy_(self._samples)

    def learn_from_replay(self, replay, updates=1):
        """``updates`` learner updates fed by ``replay.sample_device``: one CUDA graph (the same launches eagerly when
        graphs are off), then ONE read-back.  Returns the statistics of the last update.  The target copies run on the
        device, gated by a sample counter that starts from ``target_update_samples`` and is read back into it.  An
        out-of-range action in any sampled batch raises AssertionError after the read-back; that update and every later
        one of the call changed nothing."""
        K = int(updates)
        assert K >= 1
        self.current_iteration += K
        with self.total_learn_time.time():
            self._samples.fill_(self.target_update_samples)
            with self.forward_time.time():
                if self.use_cuda_graph:
                    key = (id(replay), K)
                    if key not in self._replay_graphs:
                        self._replay_graphs[key] = (ops.GraphRunner(), replay)
                    self._replay_graphs[key][0].run(lambda: self._replay_updates_device(replay, K))
                else:
                    self._replay_updates_device(replay, K)
            rb = self._readback.cpu().numpy()
            self.target_update_samples = int(rb[9])
            if self.check_action_range and rb[8] != 0:
                raise AssertionError('actions outside the integers [0, %d) (dqn.py:48)' % self.n_actions)
            stats = self._statistics(rb[0:8], hasattr(replay, 'update_priorities_device'))
            stats['performance/total_learn_time'] = self.total_learn_time.avg
            self.tensorplex.add_scalars(stats, global_step=self.current_iteration)
            self.periodic_checkpoint(global_steps=self.current_iteration, score=None)
        return stats

    def module_dict(self):
        return {'q_func': self.model}

    def checkpoint_attributes(self):
        attrs = ['current_iteration', 'model', 'model_target', 'target_update_samples']
        ck = self.session_config.checkpoint.learner
        if 'include_optimizer' in ck and ck.include_optimizer:     # extension (off by default): bit-identical continuation
            attrs += ['optim_a'] + (['optim_v'] if self.dueling else [])
        return attrs


"""DQNLearner: drop-in for surreal/learner/dqn.py:10-121 (low-dimensional observations) on hand-written kernels.

One update: the target towers (and, with double Q, the online towers) at s', the online towers at s with saved
activations, then ONE TD kernel (csrc/dqn.cu: dueling combine, argmax / gather, y = r + gamma (1 - done) q', Huber loss
weighted by the importance weights, the gradient rows of both towers, the priorities |td| + eps), the towers' backward
passes and one Adam step (eps 1e-4) over both towers with their gradient norm clipped jointly.  The target network is
copied whenever the running count of samples crosses a multiple of ``target_network_update_freq``
(PeriodicTracker.track_increment(batch_size), dqn.py:84-86)."""
import torch

from .. import _lib, ops
from .._lib import check
from .. import utils as U
from ..model.cnn_stem import joint_step
from ..model.q_net import QModel
from ..ops import _ptr
from ..session import ConfigError
from .off_policy import OffPolicyLearner

QS = dict(LOSS=0, TD_ERROR=1, Q=2, IS_WEIGHT=3, BAD_ROWS=4)
ADAM_EPS = 1e-4                                   # torch.optim.Adam(..., eps=1e-4), dqn.py:18-22


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


class DQNLearner(OffPolicyLearner):
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
        self._ta, self._tv = f(B, n), (f(B, 1) if self.dueling else None)             # target towers at s'
        self._oa, self._ov = f(B, n), (f(B, 1) if self.dueling else None)             # online towers at s' (double Q)
        self._ws = torch.zeros(_lib.lib().sb200_dqn_workspace_bytes(B), dtype=torch.uint8, device=self.device)
        self._init_off_policy(D, U.record_action_dim(self.env_config.action_spec), 8, self._ws,
                              int(_lib.lib().sb200_dqn_bad_action_offset()), counter='target_update_samples',
                              period=self.target_update_period, incr=B)
        self._stats = self._stats_block
        self.bad_action_message = 'actions outside the integers [0, %d) (dqn.py:48)' % n

    # ------------------------------------------------------------------------------------------------
    def _optimize_device(self, weights):
        """dqn.py:44-69 + _run_optimizer as one fixed launch sequence (CUDA-graph body).  ``weights`` (device [B, 1]):
        the importance weights of a prioritized batch; the rows' new priorities |td| + eps land in ``td_priorities``."""
        L, st = _lib.lib(), ops._stream()
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
        stop = self._latch_bad_action()
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

    def _target_pairs(self):
        return list(zip(self.model_target.nets(), self.model.nets()))

    def module_dict(self):
        return {'q_func': self.model}

    def checkpoint_attributes(self):
        attrs = ['current_iteration', 'model', 'model_target', 'target_update_samples']
        ck = self.session_config.checkpoint.learner
        if 'include_optimizer' in ck and ck.include_optimizer:     # extension (off by default): bit-identical continuation
            attrs += ['optim_a'] + (['optim_v'] if self.dueling else [])
        return attrs


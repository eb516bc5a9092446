"""QAgent: drop-in for surreal/agent/q_agent.py:14-87 serving a batch of actors per call.

In training every act reads epsilon = schedule(T) and then advances T (LinearSchedule from 1.0, or the PiecewiseSchedule
[(0, 1.0)] + zip(steps, final_eps)); eval_deterministic modes are greedy, other eval modes use learner_config.eval.eps.
Actor i takes the greedy argmax_j Q_j unless its draw explores, then a uniform action.  The draws come from the device's
Philox stream keyed (agent seed, T, actor) -- sb200_dqn_act_f32 -- not from CPython's ``random``.  T lives on the device,
so a replayed rollout-chunk graph advances it.  The experience wrapper is the DDPG staging with one-step records
(ExpSenderWrapperSSARNStepBootstrap, n_step = 1), whose action field holds the action index as a float."""
import ctypes as C
import time

import numpy as np
import torch

from .. import _lib, ops
from .. import utils as U
from .._lib import check
from ..env import ExpSenderWrapperSSARNStepBootstrap
from ..learner.dqn import check_dqn_config
from ..model.q_net import QModel
from .base import Agent

DETERMINISTIC_MODES = ('eval_deterministic', 'eval_deterministic_local')


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def exploration_schedule(exploration):
    """q_agent.py:67-87: LinearSchedule(steps, final_eps, 1.0), or PiecewiseSchedule([(0, 1.0)] + zip(steps, final_eps),
    outside_value=final_eps[-1])."""
    if exploration.schedule.lower() == 'linear':
        return U.LinearSchedule(schedule_timesteps=int(exploration.steps), final_p=exploration.final_eps, initial_p=1.0)
    steps, final_epses = exploration.steps, exploration.final_eps
    assert isinstance(steps, list) and isinstance(final_epses, list) and len(steps) == len(final_epses)
    return U.PiecewiseSchedule([(0, 1.0)] + list(zip(steps, final_epses)), outside_value=final_epses[-1])


class _PackedTowers:
    """PackedWeights of every tower, refreshed together at the top of a rollout chunk."""

    def __init__(self, nets):
        self.packs = [ops.PackedWeights(n) for n in nets]
        self.supported = all(p.supported for p in self.packs)

    def refresh(self):
        for p in self.packs:
            p.refresh()
        return self


class QAgent(Agent):
    def __init__(self, learner_config, env_config, session_config, agent_id, agent_mode, render=False):
        super().__init__(learner_config=learner_config, env_config=env_config, session_config=session_config,
                         agent_id=agent_id, agent_mode=agent_mode, render=render)
        if not torch.cuda.is_available():
            raise RuntimeError('surreal_b200.QAgent needs a CUDA device (there is no CPU fallback)')
        check_dqn_config(self.learner_config, self.env_config)
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.sleep_time = self.env_config.sleep_time
        self.n_actions = n = int(self.env_config.action_spec.dim[0])
        lc = self.learner_config
        self.model = QModel(obs_spec=self.env_config.obs_spec, action_dim=n, fc_hidden_sizes=lc.model.fc_hidden_sizes,
                            dueling=lc.model.dueling, convs=lc.model.convs, device=self.device)
        self.exploration = exploration_schedule(lc.algo.exploration)
        self._schedule = None
        self.fixed_eps = 0.0
        if self.agent_mode == 'training':
            pts = self.exploration.device_points()
            self._schedule = torch.tensor(pts, dtype=torch.float64, device=self.device)
            self._n_points = (len(pts) - 1) // 2
        elif self.agent_mode not in DETERMINISTIC_MODES:
            self.fixed_eps = float(lc.eval.eps)
        N, D = self.num_envs, self.model.input_dim
        self._packed = _PackedTowers(self.model.nets())
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        self._adv, self._val = f(N, n), (f(N, 1) if self.model.dueling else None)
        self._action = f(N, 1)                                   # the record's action field: the index as a float
        self._one_hot = f(N, n)                                  # what the device env steps with
        self._action_i64 = torch.zeros(N, dtype=torch.int64, device=self.device)
        self._obs_dev = f(N, D)
        self._obs_pin = None
        self._act_pin = None
        self._counter = torch.zeros(1, dtype=torch.int64, device=self.device)      # T of q_agent.py:45
        self.seed = 11 + 1000003 * int(agent_id)

    @property
    def T(self):
        """Acts so far (host read: synchronises)."""
        return int(self._counter[0])

    def epsilon(self, t=None):
        """The epsilon the next act uses (training: schedule(T))."""
        if self.agent_mode != 'training':
            return self.fixed_eps
        return self.exploration.value(self.T if t is None else t)

    def _sched_args(self):
        if self._schedule is None:
            return None, 0, self.fixed_eps
        return _p(self._schedule), self._n_points, 0.0

    def act(self, obs):
        """Device observations [N, D]: (one-hot rows [N, n_actions] for the device env, action indices [N, 1] as floats
        for the records).  Host observations (numpy): int64 actions [N] (a scalar for one actor and a 1-D observation)."""
        N, D = self.num_envs, self.model.input_dim
        if self.sleep_time > 0.0:
            time.sleep(self.sleep_time)
        x = obs['low_dim']['flat_inputs'] if isinstance(obs, dict) else obs
        if not isinstance(x, torch.Tensor):
            return self._act_host(np.asarray(x))
        x = x.reshape(N, D)
        if self._in_chunk and self._packed.supported and x.stride(1) == 1:
            # inside a multi-step chunk the weights are fixed: the chunk packed them once, at its top
            ops.mlp_forward_packed(self._packed.packs[0], x, out=self._adv)
            if self.model.dueling:
                ops.mlp_forward_packed(self._packed.packs[1], x, out=self._val)
        else:
            self.model.forward_towers(x, self._adv, self._val)
        sched, P, eps = self._sched_args()
        check(_lib.lib().sb200_dqn_act_f32(_p(self._adv), self._adv.stride(0), _p(self._val), 1, N, self.n_actions, sched,
                                           P, eps, self.seed, _p(self._counter), _p(self._action), _p(self._one_hot),
                                           self._one_hot.stride(0), None, ops._stream()), 'sb200_dqn_act_f32')
        self._counter += 1
        return self._one_hot, self._action

    def _act_host(self, x):
        """act() on a HOST observation batch through sb200_dqn_act_host_f32 (H2D obs unless the wrapper already moved it
        -> tower forwards -> epsilon-greedy -> D2H int64 actions -> one sync)."""
        N, D = self.num_envs, self.model.input_dim
        obs_host, obs_dev = self._host_obs(x, D)
        if self._act_pin is None:
            self._act_pin = torch.empty(N, dtype=torch.int64, pin_memory=True)
        sched, P, eps = self._sched_args()
        vd = self.model.state_net.desc() if self.model.dueling else None
        ad = self.model.action_net.desc()
        check(_lib.lib().sb200_dqn_act_host_f32(
            C.byref(ad), C.byref(vd) if vd is not None else None, obs_host, _p(obs_dev), N, _p(self._adv), _p(self._val),
            sched, P, eps, self.seed, _p(self._counter), _p(self._action), _p(self._action_i64),
            C.c_void_p(self._act_pin.data_ptr()), ops._stream()), 'sb200_dqn_act_host_f32')
        self._counter += 1
        a = self._act_pin.numpy().copy()
        return a[0] if (N == 1 and x.ndim == 1) else a

    def module_dict(self, model=None):
        return {'q_func': self.model if model is None else model}

    def default_config(self):
        return {'model': {'convs': '_list_', 'fc_hidden_sizes': '_list_', 'dueling': '_bool_'},
                'eval': {'eps': '_float_'}}

    def get_env(self):
        from ..env import DiscreteSyntheticEnv
        ec = self.env_config
        name = ec.env_name if 'env_name' in ec else ''
        if not str(name).startswith('synthetic'):
            return super().get_env()
        D = sum(v[0] for v in ec.obs_spec['low_dim'].values())
        return DiscreteSyntheticEnv(self.num_envs, D, self.n_actions, ec.limit_episode_length,
                                    seed=int(ec.seed) if 'seed' in ec else 0)

    def prepare_env_agent(self, env):
        env = super().prepare_env_agent(env)
        return ExpSenderWrapperSSARNStepBootstrap(env, self.learner_config, self.session_config)

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
from ..staging import Staging
from .base import Agent

DETERMINISTIC_MODES = ('eval_deterministic', 'eval_deterministic_local')


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
        self._staging = Staging(self.device)
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
        N = self.num_envs
        self._packed = _PackedTowers(self.model.nets())
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        self._adv, self._val = f(N, n), (f(N, 1) if self.model.dueling else None)
        self._action = f(N, 1)                                   # the record's action field: the index as a float
        self._one_hot = f(N, n)                                  # what the device env steps with
        self._action_i64 = torch.zeros(N, dtype=torch.int64, device=self.device)
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

    def act(self, obs):
        """QAgent.act for all N actors in ONE call of sb200_dqn_agent_act_f32, host and device observations alike: [H2D] ->
        the tower forwards (packed inside a rollout chunk) -> epsilon-greedy -> [D2H, one sync].  Device observations [N, D]:
        (one-hot rows [N, n_actions] for the device env, action indices [N, 1] as floats for the records).  Host
        observations (numpy): int64 actions [N] (a scalar for one actor and a 1-D observation)."""
        N, D = self.num_envs, self.model.input_dim
        if self.sleep_time > 0.0:
            time.sleep(self.sleep_time)
        x = obs['low_dim']['flat_inputs'] if isinstance(obs, dict) else obs
        host = not isinstance(x, torch.Tensor)
        a = _lib.DQNAgentAct()
        if host:
            x = np.asarray(x)
            a.obs_host, obs_dev = self._host_obs(x, (N, D))
            a.obs, a.ld_obs = obs_dev.data_ptr(), D
            a.action_i64 = self._action_i64.data_ptr()
            a.action_host = self._staging.pinned('action', (N,), np.int64).data_ptr()
        else:
            x = x.reshape(N, D)
            if x.stride(1) != 1:
                x = x.contiguous()
            a.obs, a.ld_obs = x.data_ptr(), x.stride(0)
            a.one_hot, a.ldo = self._one_hot.data_ptr(), self._one_hot.stride(0)
            if self._in_chunk and self._packed.supported:
                # inside a multi-step chunk the weights are fixed: the chunk packed them once, at its top
                a.adv_packed = self._packed.packs[0].buf.data_ptr()
                if self.model.dueling:
                    a.value_packed = self._packed.packs[1].buf.data_ptr()
        ad = self.model.action_net.desc()
        vd = self.model.state_net.desc() if self.model.dueling else None
        a.adv_net, a.value_net = C.pointer(ad), (C.pointer(vd) if vd is not None else None)
        a.N, a.adv, a.value = N, self._adv.data_ptr(), (self._val.data_ptr() if self._val is not None else None)
        if self._schedule is not None:
            a.schedule, a.n_points = self._schedule.data_ptr(), self._n_points
        else:
            a.fixed_eps = self.fixed_eps
        a.seed, a.act_counter, a.action = self.seed, self._counter.data_ptr(), self._action.data_ptr()
        check(_lib.lib().sb200_dqn_agent_act_f32(C.byref(a), ops._stream()), 'sb200_dqn_agent_act_f32')
        self._counter += 1
        if not host:
            return self._one_hot, self._action
        act = self._staging.pinned('action', (N,), np.int64).numpy().copy()
        return act[0] if (N == 1 and x.ndim == 1) else act

    def module_dict(self, model=None):
        return {'q_func': self.model if model is None else model}

    def default_config(self):
        return {'model': {'convs': '_list_', 'fc_hidden_sizes': '_list_', 'dueling': '_bool_'},
                'eval': {'eps': '_float_'}}

    def prepare_env_agent(self, env):
        env = super().prepare_env_agent(env)
        return ExpSenderWrapperSSARNStepBootstrap(env, self.learner_config, self.session_config)

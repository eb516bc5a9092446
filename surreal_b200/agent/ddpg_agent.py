"""DDPGAgent: drop-in for surreal/agent/ddpg_agent.py:20-215 serving a batch of actors per call.

Exploration follows the reference: actor i of ``num_agents`` explores with sigma_i = max_sigma * i /
num_agents (max_sigma / 3 for a single agent; agent 0 therefore explores with sigma = 0,
ddpg_agent.py:78-83); ``act`` = clip(pi(s)) + N(0, sigma_i) then clip again (ddpg_agent.py:176-183).
``noise_type: ou_noise`` selects Ornstein-Uhlenbeck exploration (action_noise.py:22-39; float64 state per actor, reset in
pre_episode like ddpg_agent.py:205-208).  Parameter noise (off by default) is not built."""
import ctypes as C
import time

import numpy as np
import torch

from .. import _lib, ops
from .._lib import check
from ..model.ddpg_net import DDPGModel
from ..env import ExpSenderWrapperSSARNStepBootstrap
from ..session import ConfigError
from .base import Agent


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class DDPGAgent(Agent):
    def __init__(self, learner_config, env_config, session_config, agent_id, agent_mode, render=False):
        super().__init__(learner_config=learner_config, env_config=env_config, session_config=session_config,
                         agent_id=agent_id, agent_mode=agent_mode, render=render)
        if not torch.cuda.is_available():
            raise RuntimeError('surreal_b200.DDPGAgent needs a CUDA device (there is no CPU fallback)')
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.action_dim = self.env_config.action_spec.dim[0]
        self.obs_spec = self.env_config.obs_spec
        self.use_layernorm = self.learner_config.model.use_layernorm
        self.sleep_time = self.env_config.sleep_time
        ex = self.learner_config.algo.exploration
        if ex.param_noise_type is not None:
            raise NotImplementedError('parameter noise (param_noise.py) is off by default and not built')
        self.noise_type = ex.noise_type
        if self.noise_type not in ('normal', 'ou_noise'):
            raise ConfigError('Noise type {} undefined.'.format(self.noise_type))
        N = self.num_envs
        total = int(env_config.num_agents)
        ids = np.arange(N) + int(agent_id) * N
        if total == 1:
            self.sigma = np.full(N, ex.max_sigma / 3.0)
        else:
            self.sigma = ex.max_sigma * (ids.astype(np.float64) / total)
        self.gpu_ids = 'cuda:all'
        self.model = DDPGModel(obs_spec=self.obs_spec, action_dim=self.action_dim, use_layernorm=self.use_layernorm,
                               actor_fc_hidden_sizes=self.learner_config.model.actor_fc_hidden_sizes,
                               critic_fc_hidden_sizes=self.learner_config.model.critic_fc_hidden_sizes,
                               device=self.device)
        A, D = self.action_dim, self.model.input_dim
        self._sigma = torch.tensor(self.sigma, dtype=torch.float32, device=self.device)
        self._ou_state = None
        if self.noise_type == 'ou_noise':
            self.ou_theta, self.ou_dt = float(ex.theta), float(ex.dt)
            self._sigma64 = torch.tensor(self.sigma, dtype=torch.float64, device=self.device)
            self._ou_state = torch.zeros(N, A, dtype=torch.float64, device=self.device)
        self._mean = torch.zeros(N, A, device=self.device)
        self._packed = ops.PackedWeights(self.model.actor)          # per-step inference copy of the policy weights
        self._action = torch.zeros(N, A, device=self.device)
        self._obs_dev = torch.zeros(N, D, device=self.device)
        self._obs_pin = None
        self._counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.seed = 5 + 1000003 * int(agent_id)

    def act(self, obs, unit_noise=None):
        N, A, D = self.num_envs, self.action_dim, self.model.input_dim
        if self.sleep_time > 0.0:
            time.sleep(self.sleep_time)
        x = obs['low_dim']['flat_inputs'] if isinstance(obs, dict) else obs
        if not isinstance(x, torch.Tensor):
            return self._act_host(np.asarray(x), unit_noise)
        x = x.reshape(N, D)
        if self._in_chunk and self._packed.supported and x.stride(1) == 1:
            # inside a multi-step chunk the weights are fixed: the chunk packed them once, at its top
            ops.mlp_forward_packed(self._packed, x, out=self._mean)
        else:
            ops.mlp_forward(self.model.actor, x, out=self._mean)
        det = self.agent_mode in ['eval_deterministic', 'eval_deterministic_local']
        env = self.env
        counter = env.step_counter if (env is not None and hasattr(env, 'step_counter')) else self._counter
        un = None
        if unit_noise is not None:
            un = torch.as_tensor(np.asarray(unit_noise, dtype=np.float32).reshape(N, A)).to(self.device)
        if self._ou_state is not None:
            check(_lib.lib().sb200_ddpg_ou_noise_f32(_p(self._mean), A, _p(self._sigma64), _p(un), N, A, int(det),
                                                     self.seed, _p(counter), self.ou_theta, self.ou_dt,
                                                     _p(self._ou_state), _p(self._action), ops._stream()),
                  'sb200_ddpg_ou_noise_f32')
        else:
            check(_lib.lib().sb200_ddpg_noise_f32(_p(self._mean), A, _p(self._sigma), _p(un), N, A, int(det), self.seed,
                                                  _p(counter), _p(self._action), ops._stream()), 'sb200_ddpg_noise_f32')
        if counter is self._counter:
            self._counter += 1
        return self._action

    def _act_host(self, x, unit_noise):
        """act() on a HOST observation batch through sb200_ddpg_act_host_f32 (H2D obs unless the wrapper already moved it
        -> actor forward -> exploration noise -> D2H action -> one sync): numpy in, float32 numpy out."""
        N, A, D = self.num_envs, self.action_dim, self.model.input_dim
        obs_host, obs_dev = self._host_obs(x, D)
        if getattr(self, '_act_pin', None) is None:
            self._act_pin = torch.empty(N, A, dtype=torch.float32, pin_memory=True)
        det = self.agent_mode in ['eval_deterministic', 'eval_deterministic_local']
        env = self.env
        counter = env.step_counter if (env is not None and hasattr(env, 'step_counter')) else self._counter
        un = None
        if unit_noise is not None:
            un = torch.as_tensor(np.asarray(unit_noise, dtype=np.float32).reshape(N, A)).to(self.device)
        ou = self._ou_state is not None
        d = self.model.actor.desc()
        check(_lib.lib().sb200_ddpg_act_host_f32(
            C.byref(d), obs_host, _p(obs_dev), N, _p(self._mean), _p(self._sigma), _p(self._sigma64 if ou else None),
            _p(un), int(det), self.seed, _p(counter), self.ou_theta if ou else 0.0, self.ou_dt if ou else 0.0,
            _p(self._ou_state), _p(self._action), C.c_void_p(self._act_pin.data_ptr()), ops._stream()),
            'sb200_ddpg_act_host_f32')
        if counter is self._counter:
            self._counter += 1
        a = self._act_pin.numpy().copy()
        return a.reshape(-1) if (N == 1 and x.ndim == 1) else a

    def pre_episode(self):
        super().pre_episode()
        if self._ou_state is not None and self.agent_mode not in ['eval_deterministic', 'eval_deterministic_local']:
            self._ou_state.zero_()                                  # noise.reset() (ddpg_agent.py:205-208)

    def module_dict(self, model=None):
        return {'ddpg': self.model if model is None else model}

    def default_config(self):
        return {'model': {'convs': '_list_', 'actor_fc_hidden_sizes': '_list_', 'critic_fc_hidden_sizes': '_list_'}}

    def prepare_env_agent(self, env):
        env = super().prepare_env_agent(env)
        return ExpSenderWrapperSSARNStepBootstrap(env, self.learner_config, self.session_config)

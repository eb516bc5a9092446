"""DDPGAgent: drop-in for surreal/agent/ddpg_agent.py:20-215 serving a batch of actors per call.

Exploration follows the reference: actor i of ``num_agents`` explores with sigma_i = max_sigma * i /
num_agents (max_sigma / 3 for a single agent; agent 0 therefore explores with sigma = 0,
ddpg_agent.py:78-83); ``act`` = clip(pi(s)) + N(0, sigma_i) then clip again (ddpg_agent.py:176-183).
``noise_type: ou_noise`` selects Ornstein-Uhlenbeck exploration (action_noise.py:22-39; float64 state per actor, reset in
pre_episode like ddpg_agent.py:205-208).

Parameter noise (``param_noise_type`` 'normal' / 'adaptive_normal', param_noise.py:9-74): actor k acts with its own
perturbed copy of the policy, like reference agent ``agent_id * num_envs + k`` -- its own draws, its own adaptive sigma
and action distance; the act counter ``i`` is shared because all actors act together.  Each fetch loads the unperturbed
snapshot (the reference's ``original_model``) and then builds the N images on the device (sb200_ddpg_param_noise_apply_f32);
every ``act`` runs the per-actor forward over them.  Before the first fetch the actors act with the unperturbed weights.
The reference also perturbs the critic's parameters; this agent never evaluates or publishes its critic, so that
perturbation would change nothing observable and is skipped.  Like the reference (ddpg_agent.py:120-121,136-147), the
eval_deterministic modes and any other ``param_noise_type`` value run without parameter noise."""
import ctypes as C
import time

import numpy as np
import torch

from .. import _lib, ops
from .._lib import check
from ..model.ddpg_net import DDPGModel
from ..env import ExpSenderWrapperSSARNStepBootstrap
from ..ops import _ptr
from ..session import ConfigError
from ..staging import Staging
from .base import Agent


PARAM_NOISE_TYPES = ('normal', 'adaptive_normal')
PARAM_NOISE_DIST_INTERVAL = 10          # AdaptiveNormalParameterNoise(compute_dist_interval=10), param_noise.py:31


def param_noise_stride(actor_size):
    """Floats per actor image: the flat actor size rounded up to 128 bytes."""
    return (int(actor_size) + 31) // 32 * 32


class DDPGAgent(Agent):
    def __init__(self, learner_config, env_config, session_config, agent_id, agent_mode, render=False):
        super().__init__(learner_config=learner_config, env_config=env_config, session_config=session_config,
                         agent_id=agent_id, agent_mode=agent_mode, render=render)
        if not torch.cuda.is_available():
            raise RuntimeError('surreal_b200.DDPGAgent needs a CUDA device (there is no CPU fallback)')
        self.device = torch.device('cuda', torch.cuda.current_device())
        self._staging = Staging(self.device)
        self.action_dim = self.env_config.action_spec.dim[0]
        self.obs_spec = self.env_config.obs_spec
        self.use_layernorm = self.learner_config.model.use_layernorm
        self.sleep_time = self.env_config.sleep_time
        ex = self.learner_config.algo.exploration
        det = self.agent_mode in ['eval_deterministic', 'eval_deterministic_local']
        self.param_noise_type = ex.param_noise_type if (not det and ex.param_noise_type in PARAM_NOISE_TYPES) else None
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
        A = self.action_dim
        self._sigma = torch.tensor(self.sigma, dtype=torch.float32, device=self.device)
        self._ou_state = None
        if self.noise_type == 'ou_noise':
            self.ou_theta, self.ou_dt = float(ex.theta), float(ex.dt)
            self._sigma64 = torch.tensor(self.sigma, dtype=torch.float64, device=self.device)
            self._ou_state = torch.zeros(N, A, dtype=torch.float64, device=self.device)
        self._mean = torch.zeros(N, A, device=self.device)
        self._packed = None
        if self.param_noise_type is None:
            self._packed = ops.PackedWeights(self.model.actor)      # per-step inference copy of the policy weights
        else:
            self._init_param_noise(ex)
        self._action = torch.zeros(N, A, device=self.device)
        self._counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.seed = 5 + 1000003 * int(agent_id)

    def _init_param_noise(self, ex):
        N, dev, actor = self.num_envs, self.device, self.model.actor
        self.param_noise_stride = param_noise_stride(actor.size)
        self._pn_images = torch.zeros(N * self.param_noise_stride, dtype=torch.float32, device=dev)
        self._pn_sigma = torch.full((N,), float(ex.param_noise_sigma), dtype=torch.float64, device=dev)
        self._pn_adaptive = self.param_noise_type == 'adaptive_normal'
        self.param_noise_alpha = float(ex.param_noise_alpha)
        self.param_noise_target_stddev = float(ex.param_noise_target_stddev)
        self._pn_dist = torch.zeros(N, dtype=torch.float32, device=dev) if self._pn_adaptive else None
        self._pn_state = torch.zeros(2, dtype=torch.int64, device=dev) if self._pn_adaptive else None
        self._pn_fetches = 0                 # Philox counter of the perturbation draws
        self._pn_applied = False             # False until the first fetch: act with the unperturbed weights

    @property
    def param_noise_sigma(self):
        """Per-actor parameter-noise sigma [N] (float64 copy; adaptive mode changes it at every fetch)."""
        return self._pn_sigma.cpu().numpy() if self.param_noise_type is not None else None

    def apply_param_noise(self, unit_noise=None):
        """param_noise.apply on the current (unperturbed) actor weights: adaptive sigma update, then N new images.
        ``unit_noise``: injected float64 N(0,1) draws [N, actor.size] or [N, param_noise_stride] in the flat layout
        of the actor (tests); None draws from the device Philox stream.  No host synchronisation."""
        N, actor = self.num_envs, self.model.actor
        un = None
        if unit_noise is not None:
            z = np.zeros((N, self.param_noise_stride), dtype=np.float64)
            u = np.asarray(unit_noise, dtype=np.float64).reshape(N, -1)
            z[:, :u.shape[1]] = u
            un = torch.from_numpy(z).to(self.device)
        d = actor.desc()
        check(_lib.lib().sb200_ddpg_param_noise_apply_f32(
            C.byref(d), N, _ptr(self._pn_images), self.param_noise_stride, _ptr(self._pn_sigma), _ptr(un), self.seed,
            self._pn_fetches, _ptr(self._pn_dist), _ptr(self._pn_state), self.param_noise_alpha,
            self.param_noise_target_stddev, ops._stream()), 'sb200_ddpg_param_noise_apply_f32')
        self._pn_fetches += 1
        if not self._pn_applied:
            self._pn_applied = True
            self._rollout_graphs.clear()     # captured chunks read the shared weights until now

    def on_parameter_fetched(self, params, info):
        params = super().on_parameter_fetched(params, info)
        if self.param_noise_type is None:
            return params
        self._module_dict.load(params)       # the unperturbed snapshot: original_model (param_noise.py:62)
        self.apply_param_noise()
        return None                          # loaded here already

    def _pn_descs(self):
        """(image-0 descriptor, actor stride, unperturbed descriptor or None) of the per-actor forward."""
        actor = self.model.actor
        shared = actor.desc()
        if not self._pn_applied:
            return shared, 0, (shared if self._pn_adaptive else None)
        return actor.desc(self._pn_images), self.param_noise_stride, (shared if self._pn_adaptive else None)

    def act(self, obs, unit_noise=None):
        """DDPGAgent.act (ddpg_agent.py:155-184) for all N actors in ONE call of sb200_ddpg_act_f32, host and device
        observations alike: [H2D] -> the actor forward (fused, packed inside a rollout chunk, or per actor under parameter
        noise) -> exploration noise -> [D2H, one sync].  Device observations give the device action tensor; numpy in,
        float32 numpy out (1-D for one actor's 1-D observation)."""
        N, A, D = self.num_envs, self.action_dim, self.model.input_dim
        if self.sleep_time > 0.0:
            time.sleep(self.sleep_time)
        x = obs['low_dim']['flat_inputs'] if isinstance(obs, dict) else obs
        host = not isinstance(x, torch.Tensor)
        a = _lib.DDPGAct()
        if host:
            x = np.asarray(x)
            a.obs_host, obs_dev = self._host_obs(x, (N, D))
            a.obs, a.ld_obs = obs_dev.data_ptr(), D
            a.action_host = self._staging.pinned('action', (N, A)).data_ptr()
        else:
            x = x.reshape(N, D)
            if x.stride(1) != 1:
                x = x.contiguous()
            a.obs, a.ld_obs = x.data_ptr(), x.stride(0)
        if self.param_noise_type is not None:
            d, stride, shared = self._pn_descs()
            a.forward, a.actor_stride, a.dist_interval = _lib.DDPG_FWD_PER_ACTOR, stride, PARAM_NOISE_DIST_INTERVAL
            a.shared = C.pointer(shared) if shared is not None else None
            a.dist = self._pn_dist.data_ptr() if self._pn_dist is not None else None
            a.pn_state = self._pn_state.data_ptr() if self._pn_state is not None else None
        else:
            d = self.model.actor.desc()
            if self._in_chunk and self._packed.supported:
                # inside a multi-step chunk the weights are fixed: the chunk packed them once, at its top
                a.forward, a.packed = _lib.DDPG_FWD_PACKED, self._packed.buf.data_ptr()
        a.net = C.pointer(d)
        a.N, a.mean, a.action = N, self._mean.data_ptr(), self._action.data_ptr()
        a.sigma = self._sigma.data_ptr()
        if self._ou_state is not None:
            a.sigma64, a.theta, a.dt, a.ou_state = self._sigma64.data_ptr(), self.ou_theta, self.ou_dt, self._ou_state.data_ptr()
        un = None
        if unit_noise is not None:
            un = torch.as_tensor(np.asarray(unit_noise, dtype=np.float32).reshape(N, A)).to(self.device)
            a.unit_noise = un.data_ptr()
        env = self.env
        counter = env.step_counter if (env is not None and hasattr(env, 'step_counter')) else self._counter
        a.deterministic = int(self.agent_mode in ['eval_deterministic', 'eval_deterministic_local'])
        a.seed, a.step_counter = self.seed, counter.data_ptr()
        check(_lib.lib().sb200_ddpg_act_f32(C.byref(a), ops._stream()), 'sb200_ddpg_act_f32')
        if counter is self._counter:
            self._counter += 1
        if not host:
            return self._action
        act = self._staging.pinned('action', (N, A)).numpy().copy()
        return act.reshape(-1) if (N == 1 and x.ndim == 1) else act

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

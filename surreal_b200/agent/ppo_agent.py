"""PPOAgent: drop-in for surreal/agent/ppo_agent.py:15-190 serving a whole batch of actors per call.

``act(obs)`` runs the fused actor MLP for all N actors in one launch, then one sampling kernel that
applies each actor's constant exploration scale exp(noise_i) (drawn once, ppo_agent.py:57-61), samples
N(mean, std), clips to [-1, 1] and records the behaviour policy AFTER scaling (ppo_agent.py:139,149).
numpy observations (a single actor's [D] vector or an [N, D] batch) are accepted for external CPU envs."""
import ctypes as C
import time

import numpy as np
import torch

from .. import _lib, ops
from .._lib import check
from ..model.ppo_net import PPOModel, DiagGauss
from ..env import ExpSenderWrapperMultiStepMovingWindowWithInfo
from .base import Agent


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class PPOAgent(Agent):
    def __init__(self, learner_config, env_config, session_config, agent_id, agent_mode, render=False):
        super().__init__(learner_config=learner_config, env_config=env_config, session_config=session_config,
                         agent_id=agent_id, agent_mode=agent_mode, render=render)
        if not torch.cuda.is_available():
            raise RuntimeError('surreal_b200.PPOAgent needs a CUDA device (there is no CPU fallback)')
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.action_dim = self.env_config.action_spec.dim[0]
        self.obs_spec = self.env_config.obs_spec
        self.use_z_filter = self.learner_config.algo.use_z_filter
        self.init_log_sig = self.learner_config.algo.consts.init_log_sig
        self.log_sig_range = self.learner_config.algo.consts.log_sig_range
        if self.agent_mode != 'training':
            if self.agent_mode not in ['eval_deterministic_local', 'eval_stochastic_local']:
                self.agent_mode = 'eval_stochastic' if self.env_config.stochastic_eval else 'eval_deterministic'
        N = self.num_envs
        if self.agent_mode != 'training':
            self.noise = np.zeros(N)
        else:                                  # one constant per actor (ppo_agent.py:60-61)
            self.noise = np.random.uniform(low=-self.log_sig_range, high=self.log_sig_range, size=N)
        self.rnn_config = self.learner_config.algo.rnn
        self.gpu_ids = 'cuda:all'
        self.pd = DiagGauss(self.action_dim)
        self.cells = None
        pixel = bool(self.env_config.pixel_input) if 'pixel_input' in self.env_config else False
        self.model = PPOModel(obs_spec=self.obs_spec, action_dim=self.action_dim, model_config=self.learner_config.model,
                              use_cuda=True, init_log_sig=self.init_log_sig, use_z_filter=self.use_z_filter,
                              if_pixel_input=pixel, rnn_config=self.rnn_config, device=self.device)
        A, D = self.action_dim, self.model.low_dim
        self._log_noise = torch.tensor(self.noise, dtype=torch.float32, device=self.device)
        self._mean = torch.zeros(N, A, device=self.device)
        self._packed = ops.PackedWeights(self.model.actor)          # per-step inference copy of the policy weights
        self._action = torch.zeros(N, A, device=self.device)
        self._pd = torch.zeros(N, 2 * A, device=self.device)
        self._obs_dev = torch.zeros(N, D, device=self.device)
        self._obs_pin = None
        self._out_pin = None
        self._counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.seed = 2 + 1000003 * int(agent_id)

    def set_noise(self, noise):
        self.noise = np.asarray(noise, dtype=np.float64).reshape(self.num_envs)
        self._log_noise.copy_(torch.tensor(self.noise, dtype=torch.float32))

    def act(self, obs, eps=None):
        """-> action (eval) or (action, [onetime_infos, [pd]]) in training, like ppo_agent.py:151-154.
        Device observations give device results; numpy in, numpy out."""
        N, D = self.num_envs, self.model.low_dim
        if self.model.rnn_stem is not None:
            return self._act_rnn(obs, eps)
        if self.model.cnn_stem is not None:
            return self._act_pixel(obs, eps)
        x = obs
        if isinstance(obs, dict):
            xs = [obs['low_dim'][k] for k in obs['low_dim']]
            x = xs[0] if len(xs) == 1 else (torch.cat(xs, -1) if isinstance(xs[0], torch.Tensor)
                                            else np.concatenate(xs, -1))
        host = not isinstance(x, torch.Tensor)
        if host and eps is None and isinstance(x, np.ndarray):
            return self._act_host(obs, x)                          # one C call: copies, kernels, one sync
        if host:
            cached = self.env.cached_device_obs(x) if hasattr(self.env, 'cached_device_obs') else None
            if cached is not None:
                x = cached                                         # the wrapper already moved this observation
            else:
                if self._obs_pin is None:
                    self._obs_pin = torch.empty(N, D, dtype=torch.float32, pin_memory=True)
                xt = torch.from_numpy(x) if (isinstance(x, np.ndarray) and x.dtype == np.float32 and
                                             x.flags['C_CONTIGUOUS'] and x.flags['WRITEABLE']) else None
                if xt is not None and xt.is_pinned():              # observation already in pinned memory: DMA directly
                    self._obs_dev.copy_(xt.view(N, D), non_blocking=True)
                else:
                    self._obs_pin.numpy()[...] = np.asarray(x, dtype=np.float32).reshape(N, D)
                    self._obs_dev.copy_(self._obs_pin, non_blocking=True)
                x = self._obs_dev
        x = x.reshape(N, D)
        m = self.model
        if self._in_chunk and self._packed.supported and x.stride(1) == 1:
            # inside a multi-step chunk the weights are fixed: the chunk packed them once, at its top
            ops.mlp_forward_packed(self._packed, x, zf_stats=m.z_stats, zf_eps=m.z_eps, out=self._mean)
        else:
            ops.mlp_forward(m.actor, x, zf_stats=m.z_stats, zf_eps=m.z_eps, out=self._mean)
        self._sample(eps)
        return self._host_result(True, self._unbatched(obs), []) if host else self._result(self._action, self._pd, [])

    def _unbatched(self, obs):
        """One actor's observation without the batch dimension (numpy in: its results lose theirs too)."""
        return self.num_envs == 1 and np.asarray(obs['low_dim'][next(iter(obs['low_dim']))] if isinstance(obs, dict)
                                                 else obs).ndim == 1

    def _sample(self, eps):
        """The sampling kernel on self._mean: each actor's exploration scale, N(mean, std), clip, behaviour policy -- and,
        in training behind the window wrapper, this step's staging (+ its replay-slot assignment when the wrapper fuses
        launches) -- then the step counter."""
        N, A, m, env = self.num_envs, self.action_dim, self.model, self.env
        det = self.agent_mode in ['eval_deterministic', 'eval_deterministic_local']
        staged = self.agent_mode == 'training' and isinstance(env, ExpSenderWrapperMultiStepMovingWindowWithInfo)
        counter = env.step_counter if (env is not None and hasattr(env, 'step_counter')) else self._counter
        eps_dev = None
        if eps is not None:
            eps_dev = torch.as_tensor(np.asarray(eps, dtype=np.float32).reshape(N, A)).to(self.device)
        assign = self._assign_slots(staged, counter)
        check(_lib.lib().sb200_ppo_sample_f32(
            _p(self._mean), A, _p(m.log_var), _p(self._log_noise), _p(eps_dev), N, A, int(det), self.seed, _p(counter),
            _p(self._action), _p(self._pd), C.byref(env.windows) if staged else None, int(assign), ops._stream()),
            'sb200_ppo_sample_f32')
        self._count_step(staged, counter)

    def _assign_slots(self, staged, counter):
        """Whether this step's sampling launch also assigns the step's replay slots and advances the wrapper's step
        counter (the wrapper's step() then skips its own assignment pass)."""
        assign = staged and counter is not self._counter and self.env.fuse_launches
        if assign:
            self.env.mark_slots_assigned()
        return assign

    def _count_step(self, staged, counter):
        """Advance the agent's own step counter (the seed of the sampling noise); the wrapper's advances on the device."""
        if not staged and counter is self._counter:
            self._counter += 1

    def _pinned_out(self):
        if self._out_pin is None:
            N, A = self.num_envs, self.action_dim
            self._out_pin = (torch.empty(N, A, dtype=torch.float32, pin_memory=True),
                             torch.empty(N, 2 * A, dtype=torch.float32, pin_memory=True))
        return self._out_pin

    def _host_result(self, d2h, single, onetime):
        """act()'s numpy result from the pinned outputs: with ``d2h`` the D2H copies of action / pd and one sync for both
        (else the C call has done them); float64 actions, as the reference hands the env (ppo_net.py:83); ``single``: one
        actor's unbatched observation gives unbatched results."""
        out = self._pinned_out()
        if d2h:
            out[0].copy_(self._action, non_blocking=True)
            out[1].copy_(self._pd, non_blocking=True)
            torch.cuda.current_stream().synchronize()
        action, pd = out[0].numpy().astype(np.float64), out[1].numpy().copy()
        if single:
            action, pd = action.reshape(-1), pd.reshape(-1)
        return self._result(action, pd, onetime)

    def _result(self, action, pd, onetime):
        """-> action (eval) or (action, [onetime_infos, [pd]]) in training (ppo_agent.py:151-154)."""
        if self.agent_mode != 'training':
            return action
        if self.env_config.sleep_time:
            time.sleep(self.env_config.sleep_time)
        return action, [onetime, [pd]]

    # -- RNN policy (the reference's default PPO config) ------------------------------------------------------------
    def _rnn_state(self):
        """LSTM cells of all N actors, zero-initialised (ppo_agent.py:84-93), held as torch holds them: ``_hs`` / ``_cs``
        [L, N, H], each layer's cells one contiguous [N, H] block.  ``_h`` / ``_c`` (returned) are the same storage with
        the layer dimension dropped at one layer.  NOTE: like the reference -- whose ``reset()`` no caller ever invokes --
        the cells carry over from episode to episode."""
        if getattr(self, '_h', None) is None:
            N, H, D, L = self.num_envs, self.model.rnn_stem.H, self.model.low_dim, self.model.rnn_stem.layers
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
            self._hs, self._cs, self._hs_before, self._cs_before = z(L, N, H), z(L, N, H), z(L, N, H), z(L, N, H)
            self._h, self._c = self._hs.squeeze(0), self._cs.squeeze(0)
            self._h_before, self._c_before = self._hs_before.squeeze(0), self._cs_before.squeeze(0)
            D = self.model.rnn_stem.D                             # the LSTM's input: observation or CNN feature width
            self._xf = z(N, ops._ru(D, 4))[:, :D]
            self._rnn_bufs = self.model.rnn_stem.buffers(N, 1, save=False)
        return self._h, self._c

    def _act_rnn(self, obs, eps=None):
        """act() with the LSTM stem, for host and device observations alike through ONE call of sb200_ppo_act_rnn_f32:
        z-filter -> per layer one LSTM step from each actor's cells, updated in place -> actor head -> sampling
        (ppo_net.py:317-351, ppo_agent.py:133-149).  The cells BEFORE the step are the step's onetime_info.  Host input:
        H2D of the observation (unless the wrapper already moved it), D2H of the results and one stream sync in that call.
        Pixel input: uint8 frames [N, C, H, W] (device tensor or numpy) go through the CNN stem stage of the same call
        instead of the z-filter."""
        from ..model.lstm_stem import _sfx
        N, A, D = self.num_envs, self.action_dim, self.model.low_dim
        m, stem = self.model, self.model.rnn_stem
        self._rnn_state()
        L, H = stem.layers, stem.H
        cnn = m.cnn_stem
        x = obs
        if cnn is not None:
            x = obs['pixel']['camera0'] if isinstance(obs, dict) else obs
        elif isinstance(obs, dict):
            xs = [obs['low_dim'][k] for k in obs['low_dim']]
            x = xs[0] if len(xs) == 1 else (torch.cat(xs, -1) if isinstance(xs[0], torch.Tensor) else np.concatenate(xs, -1))
        host = not isinstance(x, torch.Tensor)
        training = self.agent_mode == 'training'
        a = _lib.PPOActRnn()
        if cnn is not None:
            # CNN stem stage of the same call: frames -> conv1 -> conv2 -> fc + ReLU -> the LSTM's input rows
            D = cnn.d_out
            if not host:
                if x.dtype != torch.uint8 or x.numel() != N * cnn.C * cnn.H * cnn.W or not x.is_cuda:
                    raise ValueError('pixel act() wants uint8 CUDA frames [%d, %d, %d, %d], got %s %s'
                                     % (N, cnn.C, cnn.H, cnn.W, x.dtype, tuple(x.shape)))
                x = x.contiguous()                               # held until the call below has been issued
                a.frames = x.data_ptr()
            else:
                cached = self.env.cached_device_obs(x) if hasattr(self.env, 'cached_device_obs') else None
                if cached is not None:                           # the wrapper already moved these frames (as words)
                    a.frames = cached.data_ptr()
                else:                                            # H2D inside the call, from pinned staging
                    if self._obs_pin is None:
                        self._obs_pin = torch.empty(N, cnn.C, cnn.H, cnn.W, dtype=torch.uint8, pin_memory=True)
                        self._frames_dev = torch.empty(N, cnn.C, cnn.H, cnn.W, dtype=torch.uint8, device=self.device)
                    self._obs_pin.numpy()[...] = np.asarray(x, dtype=np.uint8).reshape(N, cnn.C, cnn.H, cnn.W)
                    a.frames_host, a.frames = self._obs_pin.data_ptr(), self._frames_dev.data_ptr()
            a.frame_c, a.frame_h, a.frame_w = cnn.C, cnn.H, cnn.W
            a.conv_w1, a.conv_b1 = cnn.seg('w1').data_ptr(), cnn.seg('b1').data_ptr()
            a.conv_w2, a.conv_b2 = cnn.seg('w2').data_ptr(), cnn.seg('b2').data_ptr()
            fc = cnn.fc.desc()
            a.fc = C.pointer(fc)
            if getattr(self, '_stem_bufs', None) is None:
                self._stem_bufs = cnn.buffers(N)
            a.a1, a.a2 = self._stem_bufs['a1'].data_ptr(), self._stem_bufs['a2'].data_ptr()
        if host:
            if cnn is None:
                obs_host, obs_dev = self._host_obs(np.asarray(x), D)
                a.obs_host, a.obs, a.ld_obs = (obs_host.value if obs_host is not None else None), obs_dev.data_ptr(), D
            out = self._pinned_out()
            a.action_host, a.pd_host = out[0].data_ptr(), out[1].data_ptr()
            if training:
                if getattr(self, '_cells_pin', None) is None:
                    self._cells_pin = (torch.empty(L, N, H, dtype=torch.float32, pin_memory=True),
                                       torch.empty(L, N, H, dtype=torch.float32, pin_memory=True))
                a.h_before_host, a.c_before_host = self._cells_pin[0].data_ptr(), self._cells_pin[1].data_ptr()
        elif cnn is None:
            x = x.reshape(N, D)
            a.obs, a.ld_obs = x.data_ptr(), x.stride(0)
        head = m.actor.desc()
        ihs = [stem.ihs[k].desc(stem.seg('ih' + _sfx(k))) for k in range(L)]
        a.head = C.pointer(head)
        a.zf = ops.zfilter_desc(m.z_stats, m.z_eps)
        for k in range(L):
            a.ih[k] = C.pointer(ihs[k])
            hh, lay = stem.seg('hh' + _sfx(k)), stem.hhs[k].layout[0]
            a.whh[k], a.bhh[k] = hh.data_ptr() + 4 * lay['w'], hh.data_ptr() + 4 * lay['b']
        a.layers, a.N, a.D, a.H = L, N, D, H
        bufs = self._rnn_bufs
        a.xf, a.ld_xf, a.pre_x = self._xf.data_ptr(), self._xf.stride(0), bufs['pre_x'].data_ptr()
        a.h_out[0], a.ldh = bufs['h_out'].data_ptr(), bufs['h_out'].stride(0)
        if L > 1:
            a.h_out[1] = bufs['h_out1'].data_ptr()
        a.h, a.c, a.h_before, a.c_before = self._hs.data_ptr(), self._cs.data_ptr(), self._hs_before.data_ptr(), self._cs_before.data_ptr()
        det = self.agent_mode in ['eval_deterministic', 'eval_deterministic_local']
        env = self.env
        staged = training and isinstance(env, ExpSenderWrapperMultiStepMovingWindowWithInfo)
        counter = env.step_counter if (env is not None and hasattr(env, 'step_counter')) else self._counter
        eps_dev = None
        if eps is not None:
            eps_dev = torch.as_tensor(np.asarray(eps, dtype=np.float32).reshape(N, A)).to(self.device)
            a.eps = eps_dev.data_ptr()
        a.mean, a.log_var, a.log_noise = self._mean.data_ptr(), m.log_var.data_ptr(), self._log_noise.data_ptr()
        a.deterministic, a.seed, a.step_counter = int(det), self.seed, counter.data_ptr()
        a.action, a.pd = self._action.data_ptr(), self._pd.data_ptr()
        if staged:
            a.stage = C.pointer(env.windows)
        a.assign_slots = self._assign_slots(staged, counter)
        check(_lib.lib().sb200_ppo_act_rnn_f32(C.byref(a), ops._stream()), 'sb200_ppo_act_rnn_f32')
        self._count_step(staged, counter)
        if not host:
            return self._result(self._action, self._pd, [self._hs_before.transpose(0, 1), self._cs_before.transpose(0, 1)])
        onetime = None
        if training:                                                # [N, layers, H]
            onetime = [self._cells_pin[0].numpy().transpose(1, 0, 2).copy(), self._cells_pin[1].numpy().transpose(1, 0, 2).copy()]
            if N == 1:
                onetime = [onetime[0][0], onetime[1][0]]
        return self._host_result(False, N == 1, onetime)

    def _act_pixel(self, obs, eps=None):
        """act() on uint8 frames [N, C, H, W] (device tensor or numpy): CNN stem -> actor head -> sampling kernel
        (ppo_net.py:268-273,368-375; ppo_agent.py:138-149)."""
        N = self.num_envs
        m, stem = self.model, self.model.cnn_stem
        fr = obs['pixel']['camera0'] if isinstance(obs, dict) else obs
        host = not isinstance(fr, torch.Tensor)
        if host:
            if self._obs_pin is None:
                self._obs_pin = torch.empty(N, stem.C, stem.H, stem.W, dtype=torch.uint8, pin_memory=True)
                self._frames_dev = torch.empty(N, stem.C, stem.H, stem.W, dtype=torch.uint8, device=self.device)
            self._obs_pin.numpy()[...] = np.asarray(fr, dtype=np.uint8).reshape(N, stem.C, stem.H, stem.W)
            self._frames_dev.copy_(self._obs_pin, non_blocking=True)
            fr = self._frames_dev
        fr = fr.reshape(N, stem.C, stem.H, stem.W)
        if getattr(self, '_stem_bufs', None) is None:
            self._stem_bufs = stem.buffers(N)
        feat = stem.forward(fr, self._stem_bufs)
        ops.mlp_forward(m.actor, feat, out=self._mean)
        self._sample(eps)
        return self._host_result(True, False, []) if host else self._result(self._action, self._pd, [])

    def _act_host(self, obs, x):
        """act() for a HOST observation batch through sb200_ppo_act_host_f32 (H2D -> forward -> sample -> D2H -> sync
        issued back to back from C): numpy in, numpy out, same results as the generic path."""
        N, D = self.num_envs, self.model.low_dim
        m, env = self.model, self.env
        out = self._pinned_out()
        obs_host, obs_dev = self._host_obs(x, D)
        det = self.agent_mode in ['eval_deterministic', 'eval_deterministic_local']
        staged = self.agent_mode == 'training' and isinstance(env, ExpSenderWrapperMultiStepMovingWindowWithInfo)
        counter = env.step_counter if (env is not None and hasattr(env, 'step_counter')) else self._counter
        assign = self._assign_slots(staged, counter)
        d = m.actor.desc()
        zf = ops.zfilter_desc(m.z_stats, m.z_eps)
        check(_lib.lib().sb200_ppo_act_host_f32(
            C.byref(d), C.byref(zf), obs_host, _p(obs_dev), N, _p(self._mean), _p(m.log_var), _p(self._log_noise),
            int(det), self.seed, _p(counter), _p(self._action), _p(self._pd), C.byref(env.windows) if staged else None,
            int(assign), C.c_void_p(out[0].data_ptr()), C.c_void_p(out[1].data_ptr()), ops._stream()),
            'sb200_ppo_act_host_f32')
        self._count_step(staged, counter)
        return self._host_result(False, self._unbatched(obs), [])

    def rollout_chunk_supported(self):
        """True when ``steps`` consecutive act -> env.step -> staging iterations can run as one persistent rollout
        kernel: training mode, the in-tree device env behind the window wrapper, and a policy that fits the kernel's
        plan -- the MLP policy on sb200_ppo_rollout_f32, the low-dim LSTM policy on sb200_ppo_rollout_rnn_f32."""
        import os
        from ..env import SyntheticEnv
        env = self.env
        if self.agent_mode != 'training' or os.environ.get('SB200_PERSISTENT_ROLLOUT', '1') == '0':
            return False
        if self.model.cnn_stem is not None:
            return False                       # pixel policies run on the per-step launch chain
        if not isinstance(env, ExpSenderWrapperMultiStepMovingWindowWithInfo) or not env.persistent_rollout:
            return False
        if type(env.env) is not SyntheticEnv:
            return False
        if self.model.rnn_stem is not None:
            a, keep = self._rollout_rnn_args(self._rollout_args())
            return bool(_lib.lib().sb200_ppo_rollout_rnn_supported(C.byref(a)))
        d = self.model.actor.desc()
        return bool(_lib.lib().sb200_ppo_rollout_supported(C.byref(d), self.model.low_dim, self.action_dim))

    def rollout_footprint(self):
        """SMs the persistent rollout kernel holds for a whole chunk when it runs in one wave (one CTA per SM); 0 when the
        chunk takes several waves or does not run on that kernel."""
        if not self.rollout_chunk_supported():
            return 0
        n = C.c_int(0)
        _lib.ensure_device()
        a = self._rollout_args()
        if self.model.rnn_stem is not None:
            r, keep = self._rollout_rnn_args(a)
            check(_lib.lib().sb200_ppo_rollout_rnn_footprint(C.byref(r), C.byref(n)), 'sb200_ppo_rollout_rnn_footprint')
        else:
            check(_lib.lib().sb200_ppo_rollout_footprint(C.byref(a), C.byref(n)), 'sb200_ppo_rollout_footprint')
        return int(n.value)

    def _rollout_args(self, ob=None, steps=0):
        """sb200_ppo_rollout of this agent's policy, env and window wrapper; with ``ob`` (the wrapper's outbox for chunks of
        ``steps``) every buffer of a chunk.  ``net`` is the actor (the LSTM policy's head); D the env's observation width."""
        m, w = self.model, self.env
        a = _lib.PPORollout()
        d = m.actor.desc()
        a.net = C.pointer(d)
        a.N, a.D, a.A, a.T = self.num_envs, m.low_dim, self.action_dim, int(steps)
        if ob is None:
            return a
        e = w.env
        a.zf_stats = m.z_stats.data_ptr() if m.z_stats is not None else None
        a.zf_eps = float(m.z_eps)
        a.log_var, a.log_noise = m.log_var.data_ptr(), self._log_noise.data_ptr()
        a.agent_seed, a.deterministic = self.seed, 0
        a.state, a.WsT, a.WaT, a.ep_step = e.state.data_ptr(), e.WsT.data_ptr(), e.WaT.data_ptr(), e.ep_step.data_ptr()
        a.max_steps, a.env_seed = e.max_steps, e.seed + 7
        a.action, a.pd = self._action.data_ptr(), self._pd.data_ptr()
        a.obs_next, a.reward, a.done = e.obs_next.data_ptr(), e.reward.data_ptr(), e.done.data_ptr()
        a.windows = C.pointer(w.windows)           # its step counter is the env's: the wrapper shares it
        a.o_obs, a.o_act, a.o_pd = ob['o_obs'].data_ptr(), ob['o_act'].data_ptr(), ob['o_pd'].data_ptr()
        a.o_rew, a.o_done = ob['o_rew'].data_ptr(), ob['o_done'].data_ptr()
        a.ev_step, a.ev_count, a.W = ob['ev_step'].data_ptr(), ob['ev_count'].data_ptr(), ob['W']
        return a

    def _rollout_rnn_args(self, a):
        """sb200_ppo_rollout_rnn around ``a``: the LSTM stem's weights and the agent's cells.  Returns it with the
        descriptors it points to (kept alive by the caller for the duration of the call)."""
        from ..model.lstm_stem import _sfx
        stem = self.model.rnn_stem
        self._rnn_state()
        r = _lib.PPORolloutRnn()
        r.base = C.pointer(a)
        ihs = [stem.ihs[k].desc(stem.seg('ih' + _sfx(k))) for k in range(stem.layers)]
        for k in range(stem.layers):
            r.ih[k] = C.pointer(ihs[k])
            hh, lay = stem.seg('hh' + _sfx(k)), stem.hhs[k].layout[0]
            r.whh[k], r.bhh[k] = hh.data_ptr() + 4 * lay['w'], hh.data_ptr() + 4 * lay['b']
        r.layers, r.H = stem.layers, stem.H
        r.h, r.c = self._hs.data_ptr(), self._cs.data_ptr()
        r.h_before, r.c_before = self._hs_before.data_ptr(), self._cs_before.data_ptr()
        return r, (a, ihs)

    def rollout_chunk(self, steps):
        """``steps`` iterations of the actor loop (agent/base.py:244-262) in one launch + the ordered commit pass."""
        w = self.env
        ob = w.rollout_outbox(steps)
        if ob is None:
            return False
        a = self._rollout_args(ob, steps)
        L, st = _lib.lib(), ops._stream()
        if self.model.rnn_stem is not None:
            r, keep = self._rollout_rnn_args(a)
            check(L.sb200_ppo_rollout_rnn_f32(C.byref(r), st), 'sb200_ppo_rollout_rnn_f32')
            a.D = w.D                              # the records carry the cells: [obs | h | c]
        else:
            check(L.sb200_ppo_rollout_f32(C.byref(a), st), 'sb200_ppo_rollout_f32')
        check(L.sb200_ppo_rollout_commit_f32(C.byref(a), _p(ob['scratch']), st), 'sb200_ppo_rollout_commit_f32')
        return True

    def module_dict(self):
        return {'ppo': self.model}

    def default_config(self):
        return {'model': {'convs': '_list_', 'fc_hidden_sizes': '_list_'}}

    def reset(self):
        """reset of LSTM hidden and cell states (ppo_agent.py:169-183; nothing in the reference calls it)."""
        if self.model.rnn_stem is not None and getattr(self, '_h', None) is not None:
            self._hs.zero_()
            self._cs.zero_()

    def prepare_env_agent(self, env):
        env = super().prepare_env_agent(env)
        if self.model.rnn_stem is not None:
            self._rnn_state()
            return ExpSenderWrapperMultiStepMovingWindowWithInfo(env, self.learner_config, self.session_config,
                                                                 cells=(self._hs, self._cs))
        return ExpSenderWrapperMultiStepMovingWindowWithInfo(env, self.learner_config, self.session_config)

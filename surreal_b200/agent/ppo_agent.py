"""PPOAgent: drop-in for surreal/agent/ppo_agent.py:15-190 serving a whole batch of actors per call.

``act(obs)`` runs the fused actor MLP for all N actors in one launch, then one sampling kernel that
applies each actor's constant exploration scale exp(noise_i) (drawn once, ppo_agent.py:57-61), samples
N(mean, std), clips to [-1, 1] and records the behaviour policy AFTER scaling (ppo_agent.py:139,149).
numpy observations (a single actor's [D] vector or an [N, D] batch) are accepted for external CPU envs.

A discrete action_spec selects the categorical policy (model.ppo_net.Categorical): the same call samples each actor's
action from the softmax of its logits.  The per-actor exploration scale has no categorical counterpart: ``noise`` /
``set_noise`` are kept but ignored by a categorical agent."""
import ctypes as C
import time

import numpy as np
import torch

from .. import _lib, ops
from .._lib import check
from ..model.ppo_net import PPOModel, Categorical, make_pd
from ..env import ExpSenderWrapperMultiStepMovingWindowWithInfo
from ..staging import Staging
from .base import Agent


class PPOAgent(Agent):
    def __init__(self, learner_config, env_config, session_config, agent_id, agent_mode, render=False):
        super().__init__(learner_config=learner_config, env_config=env_config, session_config=session_config,
                         agent_id=agent_id, agent_mode=agent_mode, render=render)
        if not torch.cuda.is_available():
            raise RuntimeError('surreal_b200.PPOAgent needs a CUDA device (there is no CPU fallback)')
        self.device = torch.device('cuda', torch.cuda.current_device())
        self._staging = Staging(self.device)
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
        self.pd = make_pd(self.env_config.action_spec)
        self.categorical = isinstance(self.pd, Categorical)
        self.cells = None
        pixel = bool(self.env_config.pixel_input) if 'pixel_input' in self.env_config else False
        self.model = PPOModel(obs_spec=self.obs_spec, action_dim=self.action_dim, model_config=self.learner_config.model,
                              use_cuda=True, init_log_sig=self.init_log_sig, use_z_filter=self.use_z_filter,
                              if_pixel_input=pixel, rnn_config=self.rnn_config, device=self.device,
                              categorical=self.categorical)
        A = self.action_dim
        self._log_noise = torch.tensor(self.noise, dtype=torch.float32, device=self.device)
        self._mean = torch.zeros(N, A, device=self.device)
        self._packed = ops.PackedWeights(self.model.actor)          # per-step inference copy of the policy weights
        self._action = torch.zeros(N, A, device=self.device)
        self._pd = torch.zeros(N, 2 * A, device=self.device)
        self._counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.seed = 2 + 1000003 * int(agent_id)

    def set_noise(self, noise):
        self.noise = np.asarray(noise, dtype=np.float64).reshape(self.num_envs)
        self._log_noise.copy_(torch.tensor(self.noise, dtype=torch.float32))

    def act(self, obs, eps=None):
        """-> action (eval) or (action, [onetime_infos, [pd]]) in training, like ppo_agent.py:151-154, through ONE call of
        sb200_ppo_act_f32 for every policy form (MLP, CNN, LSTM, CNN + LSTM) and for host and device observations alike:
        [H2D] -> [CNN stem] -> [z-filter -> LSTM layers, each actor's cells updated in place] -> actor head -> sampling
        (ppo_net.py:268-279,317-351,368-375, ppo_agent.py:133-149) -> [D2H, one sync].  The LSTM policy's onetime_infos are
        its cells BEFORE the step.  Device observations give device results; numpy in, numpy out.  Pixel input is uint8
        frames [N, C, H, W] (device tensor or numpy).  The categorical policy's action is one-hot rows [N, K] for device
        observations (what DiscreteSyntheticEnv.step takes) and int64 indices for host ones; ``eps`` is Gaussian only."""
        from ..model.lstm_stem import _sfx
        N, A, m = self.num_envs, self.action_dim, self.model
        cnn, stem = m.cnn_stem, m.rnn_stem
        if cnn is not None:
            x = obs['pixel']['camera0'] if isinstance(obs, dict) else obs
        elif isinstance(obs, dict):
            xs = [obs['low_dim'][k] for k in obs['low_dim']]
            x = xs[0] if len(xs) == 1 else (torch.cat(xs, -1) if isinstance(xs[0], torch.Tensor) else np.concatenate(xs, -1))
        else:
            x = obs
        host = not isinstance(x, torch.Tensor)
        training = self.agent_mode == 'training'
        a = _lib.PPOAct()
        D, xf = m.low_dim, None
        if cnn is not None:
            # CNN stem stage of the same call: frames -> conv1 -> conv2 -> fc + ReLU -> the LSTM's or the head's input rows
            D, shape = cnn.d_out, (N, cnn.C, cnn.H, cnn.W)
            if host:
                a.frames_host, frames = self._host_obs(np.asarray(x), shape, np.uint8)
            else:
                if x.dtype != torch.uint8 or x.numel() != N * cnn.C * cnn.H * cnn.W or not x.is_cuda:
                    raise ValueError('pixel act() wants uint8 CUDA frames [%d, %d, %d, %d], got %s %s'
                                     % (N, cnn.C, cnn.H, cnn.W, x.dtype, tuple(x.shape)))
                frames = x = x.contiguous()                      # held until the call below has been issued
            a.frames = frames.data_ptr()
            a.frame_c, a.frame_h, a.frame_w = cnn.C, cnn.H, cnn.W
            a.conv_w1, a.conv_b1 = cnn.seg('w1').data_ptr(), cnn.seg('b1').data_ptr()
            a.conv_w2, a.conv_b2 = cnn.seg('w2').data_ptr(), cnn.seg('b2').data_ptr()
            fc = cnn.fc.desc()
            a.fc = C.pointer(fc)
            if getattr(self, '_stem_bufs', None) is None:
                self._stem_bufs = cnn.buffers(N)
            a.a1, a.a2 = self._stem_bufs['a1'].data_ptr(), self._stem_bufs['a2'].data_ptr()
            xf = self._stem_bufs['feat']
        elif host:
            a.obs_host, obs_dev = self._host_obs(np.asarray(x), (N, D))
            a.obs, a.ld_obs = obs_dev.data_ptr(), D
        else:
            x = x.reshape(N, D)
            if x.stride(1) != 1:
                x = x.contiguous()
            a.obs, a.ld_obs = x.data_ptr(), x.stride(0)
            if stem is None and self._in_chunk and self._packed.supported:
                a.head_packed = self._packed.buf.data_ptr()      # weights are fixed inside a chunk: packed at its top
        if stem is not None:
            self._rnn_state()
            L, H = stem.layers, stem.H
            ihs = [stem.ihs[k].desc(stem.seg('ih' + _sfx(k))) for k in range(L)]
            for k in range(L):
                a.ih[k] = C.pointer(ihs[k])
                hh, lay = stem.seg('hh' + _sfx(k)), stem.hhs[k].layout[0]
                a.whh[k], a.bhh[k] = hh.data_ptr() + 4 * lay['w'], hh.data_ptr() + 4 * lay['b']
            a.layers, a.H = L, H
            bufs = self._rnn_bufs
            a.pre_x = bufs['pre_x'].data_ptr()
            a.h_out[0], a.ldh = bufs['h_out'].data_ptr(), bufs['h_out'].stride(0)
            if L > 1:
                a.h_out[1] = bufs['h_out1'].data_ptr()
            a.h, a.c, a.h_before, a.c_before = self._hs.data_ptr(), self._cs.data_ptr(), self._hs_before.data_ptr(), self._cs_before.data_ptr()
            xf = self._xf
        if xf is not None:
            a.xf, a.ld_xf = xf.data_ptr(), xf.stride(0)
        if host:
            st = self._staging
            a.action_host, a.pd_host = st.pinned('action', (N, A)).data_ptr(), st.pinned('pd', (N, 2 * A)).data_ptr()
            if training and stem is not None:
                a.h_before_host = st.pinned('h_before', (L, N, H)).data_ptr()
                a.c_before_host = st.pinned('c_before', (L, N, H)).data_ptr()
        head = m.actor.desc()
        a.head = C.pointer(head)
        a.zf = ops.zfilter_desc(m.z_stats, m.z_eps)
        a.N, a.D = N, D
        det = self.agent_mode in ['eval_deterministic', 'eval_deterministic_local']
        env = self.env
        staged = training and isinstance(env, ExpSenderWrapperMultiStepMovingWindowWithInfo)
        counter = env.step_counter if (env is not None and hasattr(env, 'step_counter')) else self._counter
        eps_dev = None
        a.pd_type = self.pd.pd_type
        a.mean = self._mean.data_ptr()
        if self.categorical:
            if eps is not None:
                raise ValueError('eps (injected N(0,1) draws) belongs to the Gaussian policy')
        else:
            if eps is not None:
                eps_dev = torch.as_tensor(np.asarray(eps, dtype=np.float32).reshape(N, A)).to(self.device)
                a.eps = eps_dev.data_ptr()
            a.log_var, a.log_noise = m.log_var.data_ptr(), self._log_noise.data_ptr()
        a.deterministic, a.seed, a.step_counter = int(det), self.seed, counter.data_ptr()
        a.action, a.pd = self._action.data_ptr(), self._pd.data_ptr()
        if staged:
            a.stage = C.pointer(env.windows)
        a.assign_slots = self._assign_slots(staged, counter)
        check(_lib.lib().sb200_ppo_act_f32(C.byref(a), ops._stream()), 'sb200_ppo_act_f32')
        self._count_step(staged, counter)
        if stem is None:                                            # the CNN policy keeps the batch dimension
            return self._host_result(cnn is None and self._unbatched(obs), []) if host else \
                self._result(self._action, self._pd, [])
        if not host:
            return self._result(self._action, self._pd, [self._hs_before.transpose(0, 1), self._cs_before.transpose(0, 1)])
        onetime = None
        if training:                                                # [N, layers, H]
            onetime = [self._staging.pinned(k, (L, N, H)).numpy().transpose(1, 0, 2).copy()
                       for k in ('h_before', 'c_before')]
            if N == 1:
                onetime = [onetime[0][0], onetime[1][0]]
        return self._host_result(N == 1, onetime)

    def _unbatched(self, obs):
        """One actor's observation without the batch dimension (numpy in: its results lose theirs too)."""
        return self.num_envs == 1 and np.asarray(obs['low_dim'][next(iter(obs['low_dim']))] if isinstance(obs, dict)
                                                 else obs).ndim == 1

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

    def _host_result(self, single, onetime):
        """act()'s numpy result from the pinned outputs the C call has filled: float64 actions, as the reference hands the
        env (ppo_net.py:83); ``single``: one actor's unbatched observation gives unbatched results."""
        N, A = self.num_envs, self.action_dim
        action = self._staging.pinned('action', (N, A)).numpy()
        # categorical: the index of each one-hot row; Gaussian: float64 actions
        action = action.argmax(axis=1).astype(np.int64) if self.categorical else action.astype(np.float64)
        pd = self._staging.pinned('pd', (N, 2 * A)).numpy().copy()
        if single:
            action, pd = (action[0] if self.categorical else action.reshape(-1)), pd.reshape(-1)
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

    def rollout_chunk_supported(self):
        """True when ``steps`` consecutive act -> env.step -> staging iterations can run as one persistent rollout
        kernel: training mode, the in-tree device env behind the window wrapper, and a policy that fits the kernel's
        plan -- the MLP policy on sb200_ppo_rollout_f32, the low-dim LSTM policy on sb200_ppo_rollout_rnn_f32.  The
        categorical policy takes the per-step path."""
        import os
        from ..env import SyntheticEnv
        env = self.env
        if self.agent_mode != 'training' or os.environ.get('SB200_PERSISTENT_ROLLOUT', '1') == '0':
            return False
        if self.categorical:
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
        ``steps``) every buffer of a chunk.  ``net`` is the actor (the LSTM policy's head); D the env's observation width;
        ``env`` the env's own descriptor."""
        m, w = self.model, self.env
        a = _lib.PPORollout()
        d = m.actor.desc()
        a.net = C.pointer(d)
        a.N, a.D, a.A, a.T = self.num_envs, m.low_dim, self.action_dim, int(steps)
        a.env = C.pointer(w.env.desc)
        if ob is None:
            return a
        a.zf_stats = m.z_stats.data_ptr() if m.z_stats is not None else None
        a.zf_eps = float(m.z_eps)
        a.log_var, a.log_noise = m.log_var.data_ptr(), self._log_noise.data_ptr()
        a.agent_seed, a.deterministic = self.seed, 0
        a.action, a.pd = self._action.data_ptr(), self._pd.data_ptr()
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
        check(L.sb200_ppo_rollout_commit_f32(C.byref(a), ops._ptr(ob['scratch']), st), 'sb200_ppo_rollout_commit_f32')
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

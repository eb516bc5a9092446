"""Batched HOST environments (numpy in / numpy out) driving the default agents: RNN-mode PPO at any rnn_layer and DDPG
(normal and OU noise).  One C call per act() and per wrapper step; the records staged in HBM must be bit-identical to what
the same stream produces through a device env, and match the reference's goldens."""
import copy
import tempfile

import numpy as np
import pytest
import torch

from helpers import ppo_configs, ddpg_configs, ref_state_dict
from oracle.windowing import ssar_nstep

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


class Stream:
    """Pre-generated stream of N actors over T steps: observations, successors, rewards, dones.  Actor i's episodes last
    lens[i] steps (staggered, so that episode ends cut windows mid-way); where an episode ends the next observation is a
    fresh reset draw that differs from the successor.  In a step where no actor ends, the successor IS the next
    observation (the same object, as envs without resets return it)."""

    def __init__(self, N, D, T, seed, lens=None):
        rng = np.random.default_rng(seed)
        self.N, self.D, self.T = N, D, T
        lens = np.asarray(lens if lens is not None else 6 + (np.arange(N) * 7) % 6)
        self.obs = [rng.standard_normal((N, D)).astype(np.float32)]
        self.nxt, self.rew, self.done = [], [], []
        t_ep = np.zeros(N, dtype=np.int64)
        for _ in range(T):
            t_ep += 1
            d = t_ep >= lens
            t_ep[d] = 0
            succ = rng.standard_normal((N, D)).astype(np.float32)
            if d.any():
                self.obs.append(np.where(d[:, None], rng.standard_normal((N, D)).astype(np.float32), succ))
            else:
                self.obs.append(succ)
            self.nxt.append(succ)
            self.rew.append(rng.standard_normal(N).astype(np.float32))
            self.done.append(d.astype(np.float32))


class NumpyEnv:
    """Host env replaying a Stream; rewards as float64 (as gym returns them) when rew64."""

    def __init__(self, s, A, rew64=False):
        self.s, self.N, self.D, self.A, self.rew64 = s, s.N, s.D, A, rew64
        self.t = 0

    def reset(self):
        self.t = 0
        return {'low_dim': {'flat_inputs': self.s.obs[0]}}, {}

    def step(self, action):
        assert isinstance(action, np.ndarray) and action.size == self.N * self.A
        s, t = self.s, self.t
        self.t += 1
        r = s.rew[t].astype(np.float64) if self.rew64 else s.rew[t]
        return {'low_dim': {'flat_inputs': s.obs[t + 1]}}, r, s.done[t], {'obs_next': s.nxt[t]}


class TorchEnv:
    """Device twin of NumpyEnv: the same stream as CUDA tensors (same object identities)."""

    def __init__(self, s, A):
        self.s, self.N, self.D, self.A = s, s.N, s.D, A
        self.device = torch.device(DEV)
        self.obs = [torch.tensor(o, device=DEV) for o in s.obs]
        self.nxt = [self.obs[t + 1] if s.nxt[t] is s.obs[t + 1] else torch.tensor(s.nxt[t], device=DEV) for t in range(s.T)]
        self.rew = [torch.tensor(r, device=DEV) for r in s.rew]
        self.done = [torch.tensor(d, device=DEV) for d in s.done]
        self.t = 0

    def reset(self):
        self.t = 0
        return {'low_dim': {'flat_inputs': self.obs[0]}}, {}

    def step(self, action):
        assert isinstance(action, torch.Tensor)
        t = self.t
        self.t += 1
        return {'low_dim': {'flat_inputs': self.obs[t + 1]}}, self.rew[t], self.done[t], {'obs_next': self.nxt[t]}


def _rnn_configs(D, A, H, layers, N, n_step=6, stride=4, B=4, memory_size=None, actor_h=(32, 24), critic_h=(32, 24)):
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=actor_h, critic_h=critic_h, n_step=n_step, stride=stride, B=B,
                             memory_size=memory_size)
    lc.algo.rnn.if_rnn_policy = True
    lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = 2, H, layers
    ec.num_envs = N
    return lc, ec, sc


def _ppo_host(a, N, A, L, H):
    """Host act() results normalised to torch [N, A] / [N, 2A] / [N, L, H]."""
    action, info = a
    assert isinstance(action, np.ndarray) and action.dtype == np.float64
    h, c = info[0]
    return [torch.from_numpy(action.astype(np.float32).reshape(N, A)), torch.from_numpy(info[1][0].reshape(N, 2 * A)),
            torch.from_numpy(np.ascontiguousarray(h).reshape(N, L, H)), torch.from_numpy(np.ascontiguousarray(c).reshape(N, L, H))]


def _ppo_dev(a):
    action, info = a
    return [action.cpu().clone(), info[1][0].cpu().clone(), info[0][0].cpu().clone(), info[0][1].cpu().clone()]


@pytest.mark.parametrize('layers', [1, 2])
@pytest.mark.parametrize('N', [1, 7, 256])
def test_rnn_host_env_matches_device_env_bitwise(layers, N):
    """The same observation / reward / done stream through a numpy env and through its device twin, with identical
    weights, z-filter statistics, per-actor noise and seed: every step's action, pd and onetime cells are identical, and so
    are the FIFO's control state and contents (observation rows with their cell columns, act / pd / rew / done, order and
    drops), through an agent.reset() in mid-run.  An eval_deterministic act() gives the same action on both paths."""
    from surreal_b200.agent import PPOAgent
    from surreal_b200.replay import FIFOReplay
    D, A, H, T, reset_at = 13, 3, 24, 40, 17
    s = Stream(N, D, T, seed=N + 10 * layers)
    runs, sd = [], None
    for host in (True, False):
        lc, ec, sc = _rnn_configs(D, A, H, layers, N, memory_size=max(4, N))
        R = FIFOReplay(lc, ec, sc)
        ag = PPOAgent(lc, ec, sc, 0, 'training')
        if sd is None:
            gen = torch.Generator(device=DEV).manual_seed(N)
            ag.model.z_stats.copy_(torch.cat([torch.randn(D, generator=gen, device=DEV) * 30,
                                              300 * (1.5 + torch.rand(D, generator=gen, device=DEV)),
                                              torch.tensor([300.0], device=DEV)]))
            sd = {k: v.clone() for k, v in ag.model.state_dict().items()}
        else:
            ag.model.load_state_dict(sd)
        ag.set_noise(np.linspace(-0.4, 0.4, N))
        env = NumpyEnv(s, A) if host else TorchEnv(s, A)
        ag.env = w = ag.prepare_env_agent(env)
        assert w.replay is R and w.host_env == host
        obs, _ = w.reset()
        steps = []
        for t in range(T):
            if t == reset_at:
                ag.reset()
            a = ag.act(obs)
            steps.append(_ppo_host(a, N, A, layers, H) if host else _ppo_dev(a))
            obs, _, _, _ = w.step(a)
        torch.cuda.synchronize()
        ag.agent_mode = 'eval_deterministic'
        o = s.obs[5]
        det = ag.act(o) if host else ag.act(torch.tensor(o, device=DEV)).cpu().numpy().astype(np.float64)
        runs.append(dict(steps=steps, state=R._read_state(), det=det,
                         ring=[x.clone() for x in (R.r_obs, R.r_act, R.r_pd, R.r_rew, R.r_done)],
                         stage=[x.clone() for x in (w.stage_pos, w.stage_obs, w.stage_act, w.stage_pd, w.stage_rew, w.stage_done)]))
    h, d = runs
    for t in range(T):
        for k, (x, y) in enumerate(zip(h['steps'][t], d['steps'][t])):
            assert torch.equal(x, y), (t, ['action', 'pd', 'h', 'c'][k])
    assert h['state'] == d['state'] and h['state']['total_in'] > 0
    if N > 1:
        assert h['state']['dropped'] > 0
    for x, y in zip(h['ring'] + h['stage'], d['ring'] + d['stage']):
        assert torch.equal(x, y)
    assert float(h['ring'][0][..., D:].abs().max()) > 0.0          # the cell columns ride in the records
    assert h['det'].shape == ((A,) if N == 1 else (N, A))          # one actor: a 1-D action, as before
    np.testing.assert_array_equal(h['det'].reshape(N, A), d['det'])


@pytest.mark.parametrize('name,layers', [('ppo_act_rnn', 1), ('ppo_act_rnn2', 2)])
def test_rnn_host_act_matches_reference(golden, name, layers):
    """One actor, numpy observations through the one-call entry without injected eps: pd and the onetime cells (the cells
    BEFORE each step, reset() zeroes them) against the reference's golden."""
    from surreal_b200.agent import PPOAgent
    g = golden(name)
    Hd = int(g['rnn_hidden'])
    lc, ec, sc = _rnn_configs(11, 3, Hd, layers, 1, n_step=4, stride=4, actor_h=(32, 24), critic_h=(28, 20))
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    ag.model.load_state_dict(ref_state_dict(g.sub('model/')))
    ag.set_noise(np.array([float(g['noise'])]))
    for i in range(len(g['obs'])):
        if i == int(g['reset_at']):
            ag.reset()
        a, info = ag.act(np.asarray(g['obs'][i], dtype=np.float32))
        assert a.dtype == np.float64 and a.shape == (3,)
        assert info[0][0].shape == (layers, Hd) and info[0][1].shape == (layers, Hd)
        np.testing.assert_allclose(info[0][0], np.reshape(g['h_before'][i], (layers, Hd)), rtol=0, atol=2e-6)
        np.testing.assert_allclose(info[0][1], np.reshape(g['c_before'][i], (layers, Hd)), rtol=0, atol=2e-6)
        np.testing.assert_allclose(info[1][0], g['pds'][i], rtol=0, atol=2e-6)


class NumpyScriptedEnv:
    """Host twin of the device ScriptedEnv of test_replay_rollout_gpu: obs = the actor's global step id, float64 reward
    reward_fn(g), scripted episode ends."""

    def __init__(self, scripts, reward_fn, D=2, A=1):
        self.scripts = [list(s) for s in scripts]
        self.N, self.D, self.A = len(scripts), D, A
        self.reward_fn = reward_fn
        self.ep, self.t, self.g = [0] * self.N, [0] * self.N, [0] * self.N

    def _obs(self):
        return np.array([[float(g)] * self.D for g in self.g], dtype=np.float32)

    def reset(self):
        return {'low_dim': {'flat_inputs': self._obs()}}, {}

    def step(self, action):
        rew, done = [], []
        for i in range(self.N):
            self.t[i] += 1
            self.g[i] += 1
            rew.append(self.reward_fn(self.g[i]))
            done.append(float(self.t[i] >= self.scripts[i][self.ep[i] % len(self.scripts[i])]))
        obs_next = self._obs()
        for i in range(self.N):
            if done[i]:
                self.ep[i] += 1
                self.t[i] = 0
        return ({'low_dim': {'flat_inputs': obs_next.copy()}}, np.array(rew, dtype=np.float64), np.array(done, dtype=np.float32),
                {'obs_next': obs_next})


def _ssar_host_run(case, reward_fn):
    from surreal_b200.replay import UniformReplay
    from surreal_b200.env import ExpSenderWrapperSSARNStepBootstrap as W
    n, gamma, ep_lens = case['n_step'], case['gamma'], case['ep_lens']
    lc, ec, sc = ddpg_configs(D=2, A=1, n_step=n, memory_size=64, start=0)
    lc.algo.gamma = gamma
    R = UniformReplay(lc, ec, sc)
    env = NumpyScriptedEnv([ep_lens], reward_fn)
    w = W(env, lc, sc, replay=R)
    assert w.host_env
    w.reset()
    for _ in range(sum(ep_lens)):
        w.step(np.full((1, 1), float(env.g[0]), dtype=np.float32))
    torch.cuda.synchronize()
    assert int(w.step_counter.item()) == sum(ep_lens)               # the wrapper owns the host env's step counter
    return R


@pytest.mark.parametrize('case_id', [0, 1, 2])
def test_ssar_host_staging_matches_reference_wrapper(golden, case_id):
    """The golden SSAR cases through a numpy env on the host path: records bit-exact, as the device path requires."""
    case = golden('window_ssar').js('cases')[case_id]
    R = _ssar_host_run(case, lambda g: 0.25 * g - 3.0)
    exp = case['records']
    k = len(exp)
    assert len(R) == k
    assert R.r_obs[:k, 0].cpu().numpy().astype(int).tolist() == [e['obs'] for e in exp]
    assert R.r_obs_next[:k, 0].cpu().numpy().astype(int).tolist() == [e['obs_next'] for e in exp]
    assert R.r_act[:k, 0].cpu().numpy().tolist() == [e['action'] for e in exp]
    assert R.r_done[:k].cpu().numpy().astype(bool).tolist() == [e['done'] for e in exp]
    np.testing.assert_array_equal(R.r_rew[:k].cpu().numpy(), np.array([e['reward'] for e in exp], dtype=np.float32))


def test_ssar_host_rewards_are_summed_in_float64(golden):
    """Rewards that float32 cannot represent: each record's reward is the float64 n-step sum of the reference, rounded to
    float32 once.  Summing float32-rounded rewards instead gives a different record somewhere in these cases."""
    f64 = lambda g: 0.1 * g + 1e-9                                # noqa: E731
    f32 = lambda g: float(np.float32(f64(g)))                       # noqa: E731
    differ = 0
    for case in golden('window_ssar').js('cases'):
        R = _ssar_host_run(case, f64)
        exp = ssar_nstep(case['ep_lens'], case['n_step'], case['gamma'], f64)
        k = len(exp)
        assert len(R) == k
        want = np.array([e[3] for e in exp], dtype=np.float64).astype(np.float32)
        np.testing.assert_array_equal(R.r_rew[:k].cpu().numpy(), want)
        rounded = np.array([e[3] for e in ssar_nstep(case['ep_lens'], case['n_step'], case['gamma'], f32)]).astype(np.float32)
        differ += int((rounded != want).sum())
    assert differ >= 1


@pytest.mark.parametrize('noise', ['normal', 'ou_noise'])
def test_ddpg_host_env_matches_device_env(noise):
    """Several actors, staggered episode ends, float32-representable rewards: the numpy env and its device twin give
    identical actions every step and identical uniform-ring contents."""
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.replay import UniformReplay
    N, D, A, T = 9, 12, 4, 30
    s = Stream(N, D, T, seed=7)
    runs, sd = [], None
    for host in (True, False):
        lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=(48, 32), critic_h=(64, 48), n_step=3, memory_size=100, start=0)
        lc.algo.exploration.noise_type = noise
        ec.num_envs = N
        R = UniformReplay(lc, ec, sc)
        ag = DDPGAgent(lc, ec, sc, 0, 'training')
        if sd is None:
            sd = {k: v.clone() for k, v in ag.model.state_dict().items()}
        else:
            ag.model.load_state_dict(sd)
        env = NumpyEnv(s, A, rew64=True) if host else TorchEnv(s, A)
        ag.env = w = ag.prepare_env_agent(env)
        assert w.replay is R and w.host_env == host
        obs, _ = w.reset()
        acts = []
        for _ in range(T):
            a = ag.act(obs)
            acts.append(torch.from_numpy(a.copy()) if host else a.cpu().clone())
            obs, _, _, _ = w.step(a)
        torch.cuda.synchronize()
        runs.append(dict(acts=acts, n=len(R), ring=[x.clone() for x in (R.r_obs, R.r_obs_next, R.r_act, R.r_rew, R.r_done)]))
    h, d = runs
    assert float(h['acts'][3].abs().max()) > 0.0
    for t in range(T):
        assert torch.equal(h['acts'][t], d['acts'][t]), t
    assert h['n'] == d['n'] > 0
    for x, y in zip(h['ring'], d['ring']):
        assert torch.equal(x, y)


def _default_configs(kind):
    from surreal_b200.session import Config
    if kind == 'ppo':
        from surreal_b200.main.ppo_configs import PPO_DEFAULT_LEARNER_CONFIG as L, PPO_DEFAULT_ENV_CONFIG as E, \
            PPO_DEFAULT_SESSION_CONFIG as S
    else:
        from surreal_b200.main.ddpg_configs import DDPG_DEFAULT_LEARNER_CONFIG as L, DDPG_DEFAULT_ENV_CONFIG as E, \
            DDPG_DEFAULT_SESSION_CONFIG as S
    lc, ec, sc = (Config(copy.deepcopy(c.to_dict())) for c in (L, E, S))
    sc.folder = tempfile.mkdtemp()
    return lc, ec, sc


def test_default_ppo_config_host_env_end_to_end():
    """The UNMODIFIED default PPO config (adapt mode, LSTM(100)) driven by a numpy env through the launcher and the agent's
    own main loop: the cells the learner reads for a window are the cells the agent held at the window's first step, and
    learn() on those windows agrees with the RNN oracle."""
    from surreal_b200.launch import SurrealDefaultLauncher
    from surreal_b200.agent import PPOAgent
    from surreal_b200.learner import PPOLearner
    from surreal_b200.replay import FIFOReplay
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    from oracle.ppo_rnn import OraclePPOLearnerRNN
    from oracle.filters import ZFilter as OZ
    lc, ec, sc = _default_configs('ppo')
    assert lc.algo.rnn.if_rnn_policy and lc.algo.ppo_mode == 'adapt'
    N, D, A = 32, 17, 6
    make_synthetic_env_config(ec, N, D, A, seed=3)
    n, stride, Hh, B = lc.algo.n_step, lc.algo.stride, lc.algo.rnn.rnn_hidden, lc.replay.batch_size
    s = Stream(N, D, n + stride, seed=3, lens=np.full(N, 1000))
    la = SurrealDefaultLauncher(PPOAgent, PPOLearner, FIFOReplay, sc, ec, lc)
    agent, replay, learner = la.setup_engine(env=NumpyEnv(s, A))
    assert agent.env.host_env
    cells_at, real_act = [], agent.act

    def act(obs, *args, **kw):
        cells_at.append((agent._h.clone(), agent._c.clone()))
        return real_act(obs, *args, **kw)
    agent.act = act
    agent.main_loop(max_steps=n + stride)                          # two (overlapping) windows per actor
    torch.cuda.synchronize()
    assert len(cells_at) == n + stride and len(replay) == 2 * N == B
    sd = {k: v.cpu().clone() for k, v in learner.model.state_dict().items()}
    got, real_learn = {}, learner.learn

    def learn(batch):
        got['host'] = dict(obs=batch['obs']['low_dim']['flat_inputs'].cpu().numpy(),
                           obs_next=batch['obs_next']['low_dim']['flat_inputs'].cpu().numpy(),
                           actions=batch['actions'].cpu().numpy(), rewards=batch['rewards'].cpu().numpy(),
                           dones=batch['dones'].cpu().numpy(), pd=batch['persistent_infos'][0].cpu().numpy(),
                           h0=batch['onetime_infos'][0].cpu().numpy(), c0=batch['onetime_infos'][1].cpu().numpy())
        got['st'] = real_learn(batch)
        return got['st']
    learner.learn = learn
    learner.main_loop()
    torch.cuda.synchronize()
    h0, c0 = torch.from_numpy(got['host']['h0'][:, 0]), torch.from_numpy(got['host']['c0'][:, 0])
    assert float(h0[:N].abs().max()) == 0.0 and float(c0[:N].abs().max()) == 0.0
    assert torch.equal(h0[N:], cells_at[stride][0].cpu()) and torch.equal(c0[N:], cells_at[stride][1].cpu())
    assert float(h0[N:].abs().max()) > 0.0
    al = [(sd['actor.model.seq.%d.weight' % (2 * i)], sd['actor.model.seq.%d.bias' % (2 * i)]) for i in range(3)]
    cl = [(sd['critic.model.seq.%d.weight' % (2 * i)], sd['critic.model.seq.%d.bias' % (2 * i)]) for i in range(3)]
    lstm = {k.split('.', 1)[1]: sd[k] for k in sd if k.startswith('rnn_stem.')}
    zf = OZ(D).load(sd['z_filter.running_sum'], sd['z_filter.running_sumsq'], sd['z_filter.count'])
    O = OraclePPOLearnerRNN(al, sd['actor.log_var'].view(1, A), cl, zf, lstm, A, n, B, lc.algo.rnn.horizon, Hh, 1, ppo_mode='adapt',
                            lr_actor=lc.algo.network.lr_actor, lr_critic=lc.algo.network.lr_critic)
    st, st_o = got['st'], O.learn(got['host'])
    assert learner.last_n_policy_epochs == O.n_policy_epochs[-1]
    assert float((learner._adv.cpu() - O.last_adv).abs().max()) <= 1e-5
    for k in ('_surr_loss', '_kl_loss_adapt', '_pol_kl', '_val_loss', '_entropy', '_avg_return_targ', '_avg_is_weight'):
        assert abs(st[k] - st_o[k]) <= 1e-5 * max(1.0, abs(st_o[k])), (k, st[k], st_o[k])


def test_default_ddpg_config_host_env_end_to_end():
    """The default DDPG config (small memory / start size) driven by a numpy env through the launcher: the replay holds
    exactly the transitions the n-step wrapper emits, and a few learner iterations give finite statistics."""
    from surreal_b200.launch import SurrealDefaultLauncher
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.learner import DDPGLearner
    from surreal_b200.replay import UniformReplay
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    lc, ec, sc = _default_configs('ddpg')
    N, D, A, T = 32, 12, 4, 30
    lc.replay.memory_size, lc.replay.sampling_start_size, lc.replay.batch_size = 2000, 100, 64
    make_synthetic_env_config(ec, N, D, A, seed=1)
    ec.num_agents = N
    lens = 6 + np.arange(N) % 9
    s = Stream(N, D, T, seed=11, lens=lens)
    la = SurrealDefaultLauncher(DDPGAgent, DDPGLearner, UniformReplay, sc, ec, lc)
    agent, replay, learner = la.setup_engine(env=NumpyEnv(s, A, rew64=True))
    assert agent.env.host_env
    agent.main_loop(max_steps=T)
    torch.cuda.synchronize()
    n = lc.algo.n_step
    emitted = 0
    for L in lens:                  # per actor: episodes of L steps, the last one cut at T; each piece emits max(0, len - n + 1)
        pieces = [L] * (T // L) + ([T % L] if T % L else [])
        emitted += sum(max(0, p - n + 1) for p in pieces)
    assert len(replay) == emitted
    for _ in range(3):
        st = learner.learn(replay.sample(lc.replay.batch_size))
        for k in ['actor_loss', 'critic_loss', 'Q_target', 'Q_policy', 'action_norm', 'rewards']:
            assert np.isfinite(st[k]), k


def test_one_call_per_step_launch_counts():
    """A host act() launches as many kernels as the device-observation act(): the MLP policy 2 (head, sample-assign), the
    RNN policy 2 * rnn_layer + 3 (z-filter, per layer input projection + LSTM step, head, sample-assign), the CNN policy 5
    and the CNN + LSTM policy 7 (conv1, conv2, fc in place of the z-filter); a host wrapper step launches as many
    as a device one (the commit kernel; the slots were assigned while sampling).  DDPG: 2 kernels per host act() and per
    host step.  DQN: one kernel per tower and the epsilon-greedy kernel, host and device alike."""
    from surreal_b200 import _lib
    from surreal_b200.agent import PPOAgent, DDPGAgent, QAgent
    from surreal_b200.replay import FIFOReplay, UniformReplay
    from test_pixel_rnn_gpu import _cfg as pixel_cfg
    from test_dqn_gpu import dqn_configs
    N, D, A, H = 64, 13, 3, 24

    def kernels(fn):
        torch.cuda.synchronize()
        _lib.reset_call_counter()
        r = fn()
        k = _lib.call_counter_kernels()
        torch.cuda.synchronize()
        return r, k
    for layers in (0, 1, 2):
        counts = []
        for host in (True, False):
            s = Stream(N, D, 4, seed=1)
            lc, ec, sc = _rnn_configs(D, A, H, layers, N, memory_size=4 * N)
            lc.algo.rnn.if_rnn_policy = layers > 0
            FIFOReplay(lc, ec, sc)
            ag = PPOAgent(lc, ec, sc, 0, 'training')
            ag.env = w = ag.prepare_env_agent(NumpyEnv(s, A) if host else TorchEnv(s, A))
            obs, _ = w.reset()
            a = ag.act(obs)
            obs, _, _, _ = w.step(a)                               # warm: pinned buffers and device staging exist
            a, k_act = kernels(lambda: ag.act(obs))
            _, k_step = kernels(lambda: w.step(a))
            counts.append((k_act, k_step))
        assert counts[0] == counts[1] == (2 * layers + 3 if layers else 2, 1), (layers, counts)
    for rnn, want in ((False, 5), (True, 7)):
        lc, ec, sc = pixel_cfg(2, 20, 12, A, [32, 24], [28, 20], 4, N, 'clip', 1e-4, 64, 2, 6, 1, N=N)
        lc.algo.rnn.if_rnn_policy = rnn
        ag = PPOAgent(lc, ec, sc, 0, 'training')
        fr = torch.randint(0, 256, (N, 2, 20, 20), dtype=torch.uint8)
        for obs in (fr.numpy(), fr.cuda()):
            ag.act(obs)
            assert kernels(lambda: ag.act(obs))[1] == want, (rnn, type(obs))
    for dueling in (True, False):
        lc, ec, sc = dqn_configs(D=D, dueling=dueling)
        ec.num_envs = N
        ag = QAgent(lc, ec, sc, 0, 'training')
        x = torch.randn(N, D)
        for obs in (x.numpy(), x.cuda()):
            ag.act(obs)
            assert kernels(lambda: ag.act(obs))[1] == (3 if dueling else 2), (dueling, type(obs))
    s = Stream(N, D, 4, seed=2)
    lc, ec, sc = ddpg_configs(D=D, A=A, n_step=3, memory_size=100, start=0)
    ec.num_envs = N
    UniformReplay(lc, ec, sc)
    ag = DDPGAgent(lc, ec, sc, 0, 'training')
    ag.env = w = ag.prepare_env_agent(NumpyEnv(s, A, rew64=True))
    obs, _ = w.reset()
    obs, _, _, _ = w.step(ag.act(obs))
    a, k = kernels(lambda: ag.act(obs))
    assert k == 2
    assert kernels(lambda: w.step(a))[1] == 2

"""The persistent rollout of the recurrent policy (csrc/rollout_rnn.cu, sb200_ppo_rollout_rnn_f32) and the per-step launch
chain of the same policy against float64, teacher-forced per step, and against each other.  Every record that reaches
the HBM FIFO is checked:

  (a) pd rows    == the float64 LSTM + head on the row's observation and the cells the row carries
  (b) cells      == row k+1's cells are one float64 LSTM step from row k's (the successor's and a reset row's alike)
  (c) actions    == clip(mean + std * eps, -1, 1) for the known Philox draws (keyed by the step counter)
  (d) env        == the synthetic env's dynamics on (obs, action); its draws are keyed by the step counter + 1, as the
                    chain's sampling launch advances the shared counter before the env step reads it
  (e) windows    == oracle.windowing per actor, in (completion step, actor) order through oracle.replay.FIFO

Bars: 1e-5 * max(1, rms) on pd, obs, cells and rewards, 1e-5 absolute on actions (those of test_rollout_oracle_gpu.py)."""
import numpy as np
import pytest
import torch

from helpers import ppo_configs
from oracle import nets as onets
from oracle import philox
from oracle.filters import ZFilter as OZ
from oracle.replay import FIFO as OFIFO
from test_rollout_oracle_gpu import _oracle_actor_state, _oracle_events, _ratio

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


class Case:
    """One recurrent rollout configuration (see test_rollout_oracle_gpu.Case for stagger / zf / chunks)."""

    def __init__(self, name, D, H, layers, head, A, N, n, stride, mem, L, chunks, stagger=True, zf='fit', supported=True):
        self.name, self.D, self.H, self.layers, self.head, self.A = name, D, H, layers, tuple(head), A
        self.N, self.n, self.stride, self.mem, self.L = N, n, stride, mem, L
        self.chunks, self.T = list(chunks), sum(chunks)
        self.zf, self.supported = zf, supported
        i = np.arange(N)
        self.offs = np.zeros(N, dtype=np.int64) if not stagger else ((7 * i + 3) % L if L > 0 else i % 7)


CASES = {
    # the reference's default policy: D 64, LSTM(100), head 300-200, A 8, at 1024 actors; and with 2 layers
    'default': Case('default', 64, 100, 1, (300, 200), 8, 1024, 8, 8, 8 * 1024, 40, [24, 24]),
    'default_l2': Case('default_l2', 64, 100, 2, (300, 200), 8, 256, 8, 8, 4096, 40, [24, 24], zf='edge'),
    # H a multiple of 16; N not a multiple of the 8 actors of a CTA; n != stride, windows cross chunks
    'h64_n100': Case('h64_n100', 16, 64, 1, (64, 48), 4, 100, 6, 4, 1000, 11, [9, 14], zf='edge'),
    # odd D, A = 1, odd H, one actor; the queue overflows (drop-oldest)
    'odd_n1': Case('odd_n1', 13, 37, 2, (30, 20), 1, 1, 3, 3, 4, 8, [10, 10], zf=None),
    # no episode ever ends (limit_episode_length = 0), z-filter off
    'noend': Case('noend', 20, 48, 1, (40, 24), 5, 33, 5, 5, 1000, 0, [10, 10], zf=None),
    # a 20-window queue that overflows inside one chunk
    'overflow': Case('overflow', 12, 32, 1, (32, 32), 3, 70, 4, 2, 20, 9, [7, 10]),
    # declined (H = 129 > 128): the chain runs it
    'declined': Case('declined', 16, 129, 1, (32, 32), 4, 20, 4, 4, 200, 9, [6, 6], supported=False),
}


def _setup(c, zero=False):
    """A fresh replay + RNN agent + env for case ``c``, reset, with staggered episodes.  ``zero``: every LSTM weight and the
    head's last layer zero, biases non-zero.  -> (agent, wrapper, env, replay, obs, float64 parameters)."""
    from surreal_b200.agent import PPOAgent
    from surreal_b200.replay import FIFOReplay
    from surreal_b200.env import SyntheticEnv
    D, A, N, H, Lr = c.D, c.A, c.N, c.H, c.layers
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=c.head, critic_h=(32, 32), n_step=c.n, stride=c.stride, B=N,
                             memory_size=c.mem, use_z=c.zf is not None)
    lc.algo.rnn.if_rnn_policy = True
    lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = 1, H, Lr
    ec.num_envs = N
    R = FIFOReplay(lc, ec, sc)
    ag = PPOAgent(lc, ec, sc, 3, 'training')
    g = torch.Generator().manual_seed(11)
    u = lambda k, *s: (torch.rand(*s, generator=g) * 2 - 1) * k  # noqa: E731
    w = {}
    for k in range(Lr):
        sw = 0.0 if zero else 1.5 / H ** 0.5
        w.update({'weight_ih_l%d' % k: u(sw, 4 * H, D if k == 0 else H), 'weight_hh_l%d' % k: u(sw, 4 * H, H),
                  'bias_ih_l%d' % k: u(0.3, 4 * H), 'bias_hh_l%d' % k: u(0.3, 4 * H)})
    ag.model.rnn_stem.load_torch({k: v.to(DEV) for k, v in w.items()})
    dims = [H] + list(c.head) + [A]
    layers = [(u(1.0 / np.sqrt(dims[i]), dims[i + 1], dims[i]), u(0.1, dims[i + 1])) for i in range(len(dims) - 1)]
    if zero:
        layers[-1] = (torch.zeros_like(layers[-1][0]), u(0.8, A))
    else:
        layers[-1] = (layers[-1][0] * 3, layers[-1][1])
    log_var = torch.linspace(-1.2, -0.6, A).view(1, A)
    ag.model.actor.load_layers(layers, extra=log_var)
    zf = None
    if c.zf is not None:
        zf = OZ(D)
        zf.update(torch.randn(700, D, generator=g) * 0.8 + 0.1)
        if c.zf == 'edge':
            cnt = float(zf.count)
            zf.running_sum[:4] = 0.0
            zf.running_sumsq[:2] = cnt * 1e-12
            zf.running_sumsq[2:4] = cnt * 1e-2
        ag.model.z_stats.copy_(torch.cat([zf.running_sum, zf.running_sumsq, zf.count]).to(DEV))
    noise = np.random.default_rng(5).uniform(-0.25, 0.25, N)
    ag.set_noise(noise)
    env = SyntheticEnv(N, D, A, limit_episode_length=c.L, seed=3)
    ag.env = wr = ag.prepare_env_agent(env)
    obs, _ = wr.reset()
    env.ep_step.copy_(torch.tensor(c.offs, dtype=torch.int32))
    assert ag.rollout_chunk_supported() == c.supported
    ref = dict(w={k: v.double() for k, v in w.items()}, layers=[(a.double(), b.double()) for a, b in layers],
               log_var=log_var.double(), zf=zf, noise=noise, s0=env.state.cpu().numpy().copy(), Ws=env.Ws.cpu().numpy(),
               Wa=env.Wa.cpu().numpy())
    return ag, wr, env, R, obs, ref


def _drive(c, driver, zero=False):
    ag, w, env, R, obs, ref = _setup(c, zero)
    if driver == 'step':
        for _ in range(c.T):
            obs, _, _, _ = w.step(ag.act(obs))
    else:
        for k in c.chunks:
            assert ag.rollout_chunk(k)
    torch.cuda.synchronize()
    return ag, w, env, R, ref


def _lstm64(x, h, cc, w, layers):
    """One float64 step of the stacked LSTM (torch gate order i, f, g, o): -> (h', c') [B, L, H]."""
    hs, cs = [], []
    for k in range(layers):
        gates = x @ w['weight_ih_l%d' % k].T + w['bias_ih_l%d' % k] + h[:, k] @ w['weight_hh_l%d' % k].T + w['bias_hh_l%d' % k]
        i, f, g, o = gates.chunk(4, 1)
        c1 = torch.sigmoid(f) * cc[:, k] + torch.sigmoid(i) * torch.tanh(g)
        x = torch.sigmoid(o) * torch.tanh(c1)
        hs.append(x)
        cs.append(c1)
    return torch.stack(hs, 1), torch.stack(cs, 1)


def _check_batch(c, env, ag, ref, recs, b, worst, stats):
    n, D, A, H, Lr = c.n, c.D, c.A, c.H, c.layers
    K = len(recs)
    LH = Lr * H
    actors = np.array([e[1] for e in recs])
    steps = np.array([e[2] for e in recs], dtype=np.int64)
    full = b['obs_full'].cpu().double()                                          # [K, n+1, D + 2LH]
    act, pd = b['actions'].cpu().numpy(), b['persistent_infos'][0].cpu().numpy()
    rew, done = b['rewards'].cpu().numpy(), b['dones'].cpu().numpy()
    np.testing.assert_array_equal(done, np.array([e[3] for e in recs], dtype=np.float32))
    o = full[:, :, :D]
    hc = full[:, :, D:D + LH].reshape(K, n + 1, Lr, H)
    cc = full[:, :, D + LH:].reshape(K, n + 1, Lr, H)
    x = o[:, :n].reshape(-1, D)
    if ref['zf'] is not None:
        x = ref['zf'].forward(x.float()).double()
    h1, c1 = _lstm64(x, hc[:, :n].reshape(-1, Lr, H), cc[:, :n].reshape(-1, Lr, H), ref['w'], Lr)
    # (b) the cells each successor row carries
    worst['cells'] = max(worst['cells'], _ratio(hc[:, 1:].reshape(-1, Lr, H).numpy(), h1.numpy()),
                         _ratio(cc[:, 1:].reshape(-1, Lr, H).numpy(), c1.numpy()))
    # (a) behaviour policy rows
    pdo = onets.ppo_actor(h1[:, -1], ref['layers'], ref['log_var']).numpy().reshape(K, n, 2 * A)
    pdo[:, :, A:] *= np.exp(ref['noise'])[actors, None, None]
    worst['pd'] = max(worst['pd'], _ratio(pd, pdo))
    stats['mean_max'] = max(stats['mean_max'], float(np.abs(pdo[:, :, :A]).max()))
    # (c) actions for the known draws, on the recorded and on the float64 rows
    eps = philox.agent_eps(ag.seed, steps.reshape(-1, 1), np.repeat(actors, n), A).astype(np.float64).reshape(K, n, A)
    worst['act'] = max(worst['act'], _ratio(act, np.clip(eps * pd[:, :, A:] + pd[:, :, :A], -1, 1), absolute=True),
                       _ratio(act, np.clip(eps * pdo[:, :, A:] + pdo[:, :, :A], -1, 1), absolute=True))
    stats['clipped'] += int(np.sum(np.abs(act) >= 1.0))
    stats['records'] += K
    # (d) env dynamics, draws keyed by counter + 1
    nxt, r_or = philox.synth_env_step(o[:, :n].reshape(-1, D).numpy(), act.reshape(-1, A), ref['Ws'], ref['Wa'],
                                      env.seed + 7, steps.reshape(-1, 1) + 1, np.repeat(actors, n))
    worst['obs'] = max(worst['obs'], _ratio(o[:, 1:].reshape(-1, D).numpy(), nxt))
    worst['rew'] = max(worst['rew'], _ratio(rew.reshape(-1), r_or))
    for k in range(K):                                 # the first row of an episode: the reset state
        t0, i = int(steps[k, 0]), int(actors[k])
        if t0 == 0:
            np.testing.assert_array_equal(o[k, 0].numpy(), ref['s0'][i])
            stats['resets'] += 1
        elif c.L > 0 and (t0 - (c.L - int(c.offs[i]))) % c.L == 0 and t0 >= c.L - int(c.offs[i]):
            _, _, rz = philox.env_noise(env.seed + 7, t0, [i], D)
            worst['obs'] = max(worst['obs'], _ratio(o[k, 0].numpy(), rz[0]))
            stats['resets'] += 1


def _check_run(c, driver, ag, w, env, R, ref):
    events = _oracle_events(c)
    q = OFIFO(c.mem, c.N)
    for e in events:
        q.insert(e)
    st = R._read_state()
    assert st['count'] == len(q) and st['total_in'] == len(events) and st['dropped'] == len(events) - len(q)
    assert int(env.step_counter.item()) == c.T
    pos, ep = _oracle_actor_state(c)
    np.testing.assert_array_equal(w.stage_pos.cpu().numpy(), pos)
    np.testing.assert_array_equal(env.ep_step.cpu().numpy(), ep)
    expect = list(q.q)
    worst = dict(pd=0.0, act=0.0, obs=0.0, rew=0.0, cells=0.0)
    stats = dict(clipped=0, records=0, resets=0, mean_max=0.0)
    at = 0
    while at < len(expect):
        k = min(len(expect) - at, c.mem, 1024)
        _check_batch(c, env, ag, ref, expect[at:at + k], R.sample(k), worst, stats)
        at += k
    assert stats['records'] == len(expect) > 0
    for k_, v in worst.items():
        assert v <= 1.0, '%s[%s] %s: error / bar = %.3f' % (c.name, driver, k_, v)
    assert stats['resets'] > 0
    assert (stats['mean_max'] > 0.1 and stats['clipped'] > 0) or c.N * c.A < 64     # a live head, the clip exercised
    print('%s[%s] records %d, resets %d, worst err/bar: %s' % (c.name, driver, stats['records'], stats['resets'],
                                                               ', '.join('%s %.3f' % kv for kv in worst.items())))
    return dict(state=st, pos=w.stage_pos.cpu().numpy(), ep=env.ep_step.cpu().numpy())


@pytest.mark.parametrize('name', list(CASES))
def test_rollout_rnn_matches_float64(name):
    """Both paths against float64 over the case table; the discrete state of the two paths identical."""
    c = CASES[name]
    out = [_check_run(c, d, *_drive(c, d)) for d in (['chunk', 'step'] if c.supported else ['step'])]
    if len(out) == 2:
        assert out[0]['state'] == out[1]['state']
        np.testing.assert_array_equal(out[0]['pos'], out[1]['pos'])
        np.testing.assert_array_equal(out[0]['ep'], out[1]['ep'])


def _buffers(ag, w, env, R):
    d = {k: getattr(w, k) for k in ('stage_pos', 'stage_obs', 'stage_act', 'stage_pd', 'stage_rew', 'stage_done')}
    d.update({k: getattr(R, k) for k in ('r_obs', 'r_act', 'r_pd', 'r_rew', 'r_done', 'state')})
    d.update(ep_step=env.ep_step, ctr=env.step_counter, state_env=env.state, obs_next=env.obs_next, reward=env.reward,
             done=env.done, h=ag._hs, c=ag._cs, h_before=ag._hs_before, c_before=ag._cs_before, action=ag._action,
             pd=ag._pd)
    return {k: v.clone() for k, v in d.items()}


@pytest.mark.parametrize('name', ['default', 'default_l2', 'odd_n1', 'overflow'])
def test_zero_weights_bitwise_equal_to_chain(name):
    """LSTM weights and the head's last layer zero, biases not: the two paths agree bit for bit on every buffer."""
    c = CASES[name]
    ag, w, env, R, _ = _drive(c, 'chunk', zero=True)
    p = _buffers(ag, w, env, R)
    ag, w, env, R, _ = _drive(c, 'step', zero=True)
    s = _buffers(ag, w, env, R)
    for k in p:
        assert torch.equal(p[k], s[k]), k
    assert float(p['h'].abs().max()) > 0.05 and float(p['r_obs'].abs().max()) > 0.05


def test_live_weights_close_to_chain():
    """Live weights: the discrete state of the two paths identical over 48 steps; after 8 steps the continuous state
    within 1e-4 * max(1, rms) (the two paths round differently, and the recurrence and the env carry the differences
    from step to step; each record is held to 1e-5 against float64 in test_rollout_rnn_matches_float64)."""
    c = CASES['default_l2']
    p = _buffers(*_drive(c, 'chunk')[:4])
    s = _buffers(*_drive(c, 'step')[:4])
    for k in ('stage_pos', 'ep_step', 'ctr', 'state', 'r_done', 'stage_done', 'done'):
        assert torch.equal(p[k], s[k]), k
    c = Case('short', 64, 100, 2, (300, 200), 8, 256, 8, 8, 4096, 40, [4, 4], zf='edge')
    p = _buffers(*_drive(c, 'chunk')[:4])
    s = _buffers(*_drive(c, 'step')[:4])
    for k in ('h', 'c', 'h_before', 'c_before', 'pd', 'stage_obs', 'stage_pd', 'state_env', 'reward'):
        assert _ratio(p[k].cpu().numpy(), s[k].cpu().numpy(), tol=1e-4) <= 1.0, k


def test_chunks_then_act_carry_the_cells():
    """After persistent chunks act() continues from the cells the kernel wrote back, as after the chain."""
    c = CASES['h64_n100']
    outs = []
    for d in ('chunk', 'step'):
        ag, w, env, R, _ = _drive(c, d)
        ag.act(env.state)
        torch.cuda.synchronize()
        outs.append((ag._hs_before.clone(), ag._hs.clone(), ag._pd.clone()))
    for a, b in zip(*outs):
        assert _ratio(a.cpu().numpy(), b.cpu().numpy()) <= 1.0


def test_main_loop_graph_equals_direct_chunks_and_picks_up_new_parameters():
    """main_loop's captured graph replays equal direct rollout_chunk calls bit for bit, also when the policy's parameters
    change between chunks.  The change is simulated: new values written in place, at the addresses a parameter fetch
    writes to, with no publish / fetch round trip."""
    from surreal_b200.ops import graphs_enabled
    assert graphs_enabled()
    c = Case('graph', 16, 48, 2, (40, 24), 4, 64, 6, 3, 2000, 17, [11, 11, 11])
    runs = []
    for driver in ('graph', 'chunk'):
        ag, w, env, R, obs, _ = _setup(c)
        ag._obs = obs
        for j, k in enumerate(c.chunks):
            if j == 2:                                   # simulated fetch: new values, same addresses
                ag.model.actor.params.mul_(0.5)
                ag.model.rnn_stem.params.mul_(0.5)
            if driver == 'graph':
                ag.main_loop(max_steps=k)
            else:
                assert ag.rollout_chunk(k)
        torch.cuda.synchronize()
        if driver == 'graph':
            assert list(ag._rollout_graphs) == [11] and ag._rollout_graphs[11].graph is not None
        runs.append(_buffers(ag, w, env, R))
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k


def test_env_switch_runs_the_chain(monkeypatch):
    """SB200_PERSISTENT_ROLLOUT=0: main_loop runs the per-step chain (the persistent entry is never called) and its
    records pass the float64 checks."""
    monkeypatch.setenv('SB200_PERSISTENT_ROLLOUT', '0')
    c = Case('env_off', 12, 32, 1, (32, 32), 3, 70, 4, 2, 20, 9, [17], supported=False)
    ag, w, env, R, obs, ref = _setup(c)
    assert ag.rollout_footprint() == 0
    calls = []
    monkeypatch.setattr(ag, 'rollout_chunk', lambda steps: calls.append(steps))
    ag._obs = obs
    ag.main_loop(max_steps=c.T)
    torch.cuda.synchronize()
    assert calls == []
    _check_run(c, 'env_off', ag, w, env, R, ref)


def test_footprint_and_declined_paths():
    """The footprint is the kernel's CTA count (8 actors each) while that fits one wave, 0 past it; eval mode and a
    CNN + LSTM policy take the chain."""
    ag = _setup(Case('fp', 16, 48, 1, (40, 24), 4, 256, 4, 4, 100, 9, [5]))[0]
    assert ag.rollout_footprint() == 32
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    big = _setup(Case('fp_big', 16, 48, 1, (40, 24), 4, 8 * n_sm + 1, 4, 4, 100, 9, [5]))[0]
    assert big.rollout_footprint() == 0
    ag.agent_mode = 'eval_stochastic'
    assert not ag.rollout_chunk_supported()
    from surreal_b200.agent import PPOAgent
    from surreal_b200.env import SyntheticPixelEnv
    from surreal_b200.replay import FIFOReplay
    N = 16
    lc, ec, sc = ppo_configs(D=1, A=3, actor_h=(32, 24), critic_h=(28, 20), n_step=4, stride=4, B=N, use_z=False)
    ec.obs_spec = {'pixel': {'camera0': (2, 20, 20)}}
    ec.pixel_input = True
    ec.num_envs = N
    lc.model.cnn_feature_dim = 12
    lc.algo.rnn.if_rnn_policy = True
    lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = 2, 16, 1
    FIFOReplay(lc, ec, sc)
    px = PPOAgent(lc, ec, sc, 0, 'training')
    px.env = pw = px.prepare_env_agent(SyntheticPixelEnv(N, (2, 20, 20), 3, limit_episode_length=5, seed=9))
    pw.reset()
    assert px.model.cnn_stem is not None and px.model.rnn_stem is not None
    assert not px.rollout_chunk_supported() and px.rollout_footprint() == 0


def _engine(N, layers):
    """PipelinedEngine with the LSTM policy on the synthetic env: n == stride == T, N == batch size."""
    from surreal_b200.launch import SurrealDefaultLauncher, PipelinedEngine
    from surreal_b200.agent import PPOAgent
    from surreal_b200.learner import PPOLearner
    from surreal_b200.replay import FIFOReplay
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    n = 8
    lc, ec, sc = ppo_configs(D=16, A=4, actor_h=(64, 48), critic_h=(64, 48), n_step=n, stride=n, B=N,
                             memory_size=2 * N, exp_interval=N)
    lc.algo.rnn.if_rnn_policy = True
    lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = 2, 32, layers
    make_synthetic_env_config(ec, N, 16, 4, seed=5)
    ec.limit_episode_length = 2 * n
    sc.agent.fetch_parameter_interval = n
    lc.parameter_publish.min_publish_interval = 0.0
    la = SurrealDefaultLauncher(PPOAgent, PPOLearner, FIFOReplay, sc, ec, lc)
    agent, replay, learner = la.setup_engine()
    assert agent.model.rnn_stem is not None and agent.rollout_chunk_supported()
    return agent, replay, learner, PipelinedEngine(agent, replay, learner, n)


def _run_engine(N, eng, agent, replay, learner, steps):
    eng.prime()
    versions = []
    for _ in range(steps):
        st = eng.step()
        assert st and all(np.isfinite(v) for v in st.values())
        versions.append(learner.publisher.version)
    eng.drain()
    s = replay._read_state()
    # every window consumed exactly once, oldest first: steps + 1 rollouts of N windows in, steps batches of N out
    assert s['total_in'] == (steps + 1) * N and s['total_out'] == steps * N and s['count'] == N and s['dropped'] == 0
    assert s['head'] == (steps * N) % s['capacity']
    assert versions == list(range(1, steps + 1))
    assert agent._ps_client._last_version in (steps - 1, steps)
    assert learner.current_iteration == steps


@pytest.mark.parametrize('layers', [1, 2])
def test_pipelined_engine_overlaps_the_rnn_rollout(layers):
    """PipelinedEngine with the LSTM policy: the persistent rollout holds 16 SMs, so the learner runs beside it on the
    rest; every window is consumed exactly once, in arrival order, and the learner's statistics are finite."""
    N = 128
    agent, replay, learner, eng = _engine(N, layers)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    assert agent.rollout_footprint() == N // 8 and eng.overlap and learner.sm_budget == n_sm - N // 8
    _run_engine(N, eng, agent, replay, learner, 5)


def test_pipelined_engine_without_overlap_past_one_wave():
    """Past one wave (more CTAs than SMs) the footprint is 0: no overlap, the learner's epochs wait for the rollout."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    N = 8 * n_sm + 8
    agent, replay, learner, eng = _engine(N, 1)
    assert agent.rollout_footprint() == 0 and not eng.overlap and learner.sm_budget == 0
    _run_engine(N, eng, agent, replay, learner, 2)

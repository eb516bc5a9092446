"""The persistent rollout kernel (the kernel that carries the headline number) and the per-step launch path against the
ORACLE, across the shapes, configs and drivers that select different code in the kernel.  Every record that reaches
the HBM FIFO is checked:

  (a) pd rows   == oracle.nets.ppo_actor(OZFilter.forward(obs)) with stds scaled by exp(noise_i)   (ppo_agent.py:133-139,149)
  (b) actions   == clip(mean + std * eps, -1, 1) for the known Philox draws                         (ppo_agent.py:140-145)
  (c) env       == the synthetic env's dynamics on (obs, action) with the known Philox draws (SURVEY §8d cfg 2),
                   and the first observation of an episode is the env's reset state
  (d) windows   == oracle.windowing.multistep_windows per actor (clear-on-done, tails discarded), queued in
                   (completion step, actor) arrival order through oracle.replay.FIFO               (exp_sender_wrapper.py:204-228,
                                                                                                    fifo_replay.py:27-39)
Actors start at staggered points of their episodes (env.ep_step is set after reset), so windows of different actors
complete at different steps and the commit pass has to interleave them.  The FIFO control block, the step counter and
each actor's staging position / episode step are checked too, and the persistent and per-step paths must agree on
all of these exactly.

Bars: 1e-5 * max(1, rms) on pd / obs / rewards, 1e-5 absolute on actions (|a| <= 1).  Worst measured ratio err / bar
over every case and both paths, on an H100 80GB HBM3: pd 0.085, obs 0.077, reward 0.024, actions 0.081 (pd and
actions: the per-step path at 4096 actors; obs: the persistent kernel at D = 128).  The oracle's policy forward runs
in float64 on its own float32 z-filter output."""
import numpy as np
import pytest
import torch

from helpers import ppo_configs
from oracle import nets as onets
from oracle import philox
from oracle.filters import ZFilter as OZ
from oracle.replay import FIFO as OFIFO
from oracle.windowing import multistep_windows

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SUBSET_ABOVE = 4096          # from this many actors on, the numbers are checked on a fixed subset of actors


def _ratio(got, exp, tol=1e-5, absolute=False):
    got, exp = np.asarray(got, dtype=np.float64), np.asarray(exp, dtype=np.float64)
    bar = tol if absolute else tol * max(1.0, float(np.sqrt(np.mean(exp ** 2))))
    return float(np.abs(got - exp).max()) / bar if got.size else 0.0


class Case:
    """One rollout configuration.  ``stagger``: actor i starts (off_i) steps into its first episode; ``zf``: 'fit'
    (statistics of a N(0.1, 0.8) sample), 'edge' (two dims with variance below z_eps, two with std 0.1 so that
    observations land beyond +-5) or None (z-filter off); ``chunks``: steps per rollout_chunk / main_loop call."""

    def __init__(self, name, shape, N, n, stride, mem, L, chunks, stagger=True, zf='fit', supported=True):
        self.name = name
        self.D, self.H1, self.H2, self.A = shape
        self.N, self.n, self.stride, self.mem, self.L = N, n, stride, mem, L
        self.chunks, self.T = list(chunks), sum(chunks)
        self.zf, self.supported = zf, supported
        i = np.arange(N)
        if not stagger:
            self.offs = np.zeros(N, dtype=np.int64)
        elif L > 0:
            self.offs = (7 * i + 3) % L
        else:
            self.offs = i % 7                    # no episode ever ends: the offsets only carry through ep_step
        self.subset = np.arange(N) if N < SUBSET_ABOVE else \
            np.unique(np.concatenate([np.arange(128), np.arange(N // 2, N // 2 + 32), np.arange(N - 128, N)]))


CASES = {
    # 222,224 B of shared memory; head passes n8 = 0 / 8 / 16, the last one half width; z-filter edges
    'a20_smem': Case('a20_smem', (64, 256, 256, 20), 100, 8, 8, 1000, 13, [16, 16], zf='edge'),
    # 228,128 B: the largest head that still fits the 229,376 B (224 KB) plan; n != stride, windows cross chunks
    'a24_smem_max': Case('a24_smem_max', (64, 256, 256, 24), 64, 6, 4, 1000, 11, [9, 14], zf=None),
    # 232,688 B: declined, the per-step path runs it
    'a25_declined': Case('a25_declined', (64, 256, 256, 25), 64, 6, 4, 1000, 11, [9, 14], supported=False),
    # D = 128 (the kernel's maximum), 220,480 B; n != stride
    'd128': Case('d128', (128, 176, 176, 8), 96, 5, 3, 1000, 9, [7, 11]),
    # 233,568 B: declined
    'd128_declined': Case('d128_declined', (128, 192, 192, 8), 32, 5, 3, 1000, 9, [7, 11], supported=False),
    # head_mode 0, A not a multiple of 8 (passes 0 / 8, the second half width), one actor in a second cluster; no
    # episode ever ends (limit_episode_length = 0)
    'hm0_a12_noend': Case('hm0_a12_noend', (8, 32, 32, 12), 33, 6, 6, 1000, 0, [10, 10]),
    # head_mode 0 with all 32 lanes live, z-filter off
    'hm0_a32': Case('hm0_a32', (16, 64, 64, 32), 50, 4, 4, 1000, 10, [12, 12], zf=None),
    # head_mode 0, H1 != H2, D / 4 odd (k-split tail of the first layer), z-filter edges; a 50-window queue that
    # overflows inside one chunk (drop-oldest in the commit pass)
    'hm0_h1h2_overflow': Case('hm0_h1h2_overflow', (20, 32, 48, 17), 70, 4, 2, 50, 9, [7, 10], zf='edge'),
    # one valid actor in its cluster, D / 4 odd, H / 16 = 9 and 5
    'd100_n1': Case('d100_n1', (100, 144, 80, 5), 1, 4, 3, 100, 7, [13, 8]),
    # the smallest plan: D = 4 (the upper k half of the first layer is empty), A = 1; queue overflows
    'd4_a1': Case('d4_a1', (4, 16, 16, 1), 40, 3, 3, 30, 8, [10, 10]),
    # BASELINE configs[4] per-GPU shapes at dp1 and dp8: n = 256, episode 512, one 512-step chunk
    'cfg4_dp1': Case('cfg4_dp1', (64, 256, 256, 8), 4096, 256, 256, 2 * 4096, 512, [512]),
    'cfg4_dp8': Case('cfg4_dp8', (64, 256, 256, 8), 512, 256, 256, 2 * 512, 512, [512]),
}


def _setup(c):
    """A fresh replay + agent + env for case ``c``, reset, with staggered episodes.  -> (agent, wrapper, env, replay,
    oracle-side parameters)."""
    from surreal_b200.agent import PPOAgent
    from surreal_b200.replay import FIFOReplay
    from surreal_b200.env import SyntheticEnv
    D, A, N = c.D, c.A, c.N
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=(c.H1, c.H2), critic_h=(c.H1, c.H2), n_step=c.n, stride=c.stride, B=N,
                             memory_size=c.mem, use_z=c.zf is not None)
    ec.num_envs = N
    R = FIFOReplay(lc, ec, sc)
    ag = PPOAgent(lc, ec, sc, 3, 'training')
    g = torch.Generator().manual_seed(11)
    dims = [D, c.H1, c.H2, A]
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / np.sqrt(dims[i]),
               (torch.rand(dims[i + 1], generator=g) * 2 - 1) * 0.1) for i in range(3)]
    log_var = torch.linspace(-1.2, -0.6, A).view(1, A)
    ag.model.actor.load_layers(layers, extra=log_var)
    zf = None
    if c.zf is not None:
        zf = OZ(D)
        zf.update(torch.randn(700, D, generator=g) * 0.8 + 0.1)
        if c.zf == 'edge':
            cnt = float(zf.count)
            zf.running_sum[:4] = 0.0
            zf.running_sumsq[:2] = cnt * 1e-12               # std 1e-6: floored at z_eps = 1e-5
            zf.running_sumsq[2:4] = cnt * 1e-2               # std 0.1: most observations clamp at +-5
        ag.model.z_stats.copy_(torch.cat([zf.running_sum, zf.running_sumsq, zf.count]).to(DEV))
    noise = np.random.default_rng(5).uniform(-0.25, 0.25, N)
    ag.set_noise(noise)
    env = SyntheticEnv(N, D, A, limit_episode_length=c.L, seed=3)
    ag.env = w = ag.prepare_env_agent(env)
    obs, _ = w.reset()
    env.ep_step.copy_(torch.tensor(c.offs, dtype=torch.int32))
    assert ag.rollout_chunk_supported() == c.supported
    ref = dict(layers=layers, log_var=log_var, zf=zf, noise=noise, s0=env.state.cpu().numpy().copy(),
               Ws=env.Ws.cpu().numpy(), Wa=env.Wa.cpu().numpy())
    return ag, w, env, R, obs, ref


def _drive(c, driver):
    """Run case ``c`` through 'chunk' (agent.rollout_chunk), 'step' (act / env.step per step) or 'graph'
    (agent.main_loop, CUDA-graph capture on its first call, replays after)."""
    ag, w, env, R, obs, ref = _setup(c)
    if driver == 'step':
        for _ in range(c.T):
            obs, _, _, _ = w.step(ag.act(obs))
    elif driver == 'chunk':
        for k in c.chunks:
            assert ag.rollout_chunk(k)
    else:
        from surreal_b200.ops import graphs_enabled
        assert graphs_enabled() and len(set(c.chunks)) == 1
        ag._obs = obs
        for k in c.chunks:
            ag.main_loop(max_steps=k)
        assert list(ag._rollout_graphs) == [c.chunks[0]] and ag._rollout_graphs[c.chunks[0]].graph is not None
    torch.cuda.synchronize()
    return ag, w, env, R, ref


def _oracle_events(c):
    """Every window completed within T steps as (completion step, actor, obs step ids, done flags), in arrival order."""
    per_off, events = {}, []
    for i in range(c.N):
        off = int(c.offs[i])
        if off not in per_off:
            if c.L > 0:
                lens = [c.L - off]
                while sum(lens) <= c.T:
                    lens.append(c.L)
            else:
                lens = [c.T + c.n + 1]
            per_off[off] = [(ids, dn) for ids, nxt, dn in multistep_windows(lens, c.n, c.stride) if nxt <= c.T]
        for ids, dn in per_off[off]:
            events.append((ids[-1], i, ids, dn))
    events.sort(key=lambda e: (e[0], e[1]))
    return events


def _oracle_actor_state(c):
    """(stage_pos, ep_step) of every actor after T steps: the deque length of its current episode and its step count."""
    pos, ep = np.zeros(c.N, dtype=np.int64), np.zeros(c.N, dtype=np.int64)
    for i in range(c.N):
        off = int(c.offs[i])
        if c.L > 0:
            first = c.L - off
            since = c.T if c.T < first else (c.T - first) % c.L
            ep[i] = (off + c.T) % c.L
        else:
            since, ep[i] = c.T, off + c.T
        q = 0
        for _ in range(since):
            q += 1
            if q == c.n:
                q = max(0, c.n - c.stride)
        pos[i] = q
    return pos, ep


def _episode_starts(c, actor):
    if c.L == 0:
        return {0}
    first = c.L - int(c.offs[actor])
    return {0} | set(range(first, c.T + 1, c.L))


def _check_batch(c, ag, env, ref, recs, b, worst, stats):
    """Records ``recs`` (oracle events) against the device batch ``b`` that popped them."""
    N, n, D, A = c.N, c.n, c.D, c.A
    K = len(recs)
    actors = np.array([e[1] for e in recs])
    steps = np.array([e[2] for e in recs], dtype=np.int64)                      # [K, n]
    obs_full = b['obs_full'].cpu().numpy()                                       # [K, n+1, D]
    act, pd = b['actions'].cpu().numpy(), b['persistent_infos'][0].cpu().numpy()
    rew, done = b['rewards'].cpu().numpy(), b['dones'].cpu().numpy()
    # (d) every record: done flags of its window, and its identity -- the std columns of its actor and the actions of
    # the Philox draws at its (step, actor), applied to the mean / std the record carries
    np.testing.assert_array_equal(done, np.array([e[3] for e in recs], dtype=np.float32))
    std_i = (np.exp(ref['log_var'].numpy().astype(np.float64)) * np.exp(ref['noise'])[actors, None])      # [K, A]
    np.testing.assert_allclose(pd[:, :, A:], np.broadcast_to(std_i[:, None, :], (K, n, A)), rtol=1e-6, atol=0)
    eps = philox.agent_eps(ag.seed, steps.reshape(-1, 1), np.repeat(actors, n), A).astype(np.float64).reshape(K, n, A)
    a_rec = np.clip(eps * pd[:, :, A:].astype(np.float64) + pd[:, :, :A], -1, 1)
    worst['act'] = max(worst['act'], _ratio(act, a_rec, absolute=True))
    stats['clipped'] += int(np.sum(np.abs(act) >= 1.0))
    stats['records'] += K
    # the numbers, on the subset of actors
    sel = np.isin(actors, c.subset)
    if not sel.any():
        return
    actors, steps, obs_full, act, pd, rew, eps = (v[sel] for v in (actors, steps, obs_full, act, pd, rew, eps))
    K = len(actors)
    # (a) behaviour policy rows: the float64 forward on the oracle's z-filtered observation
    x = torch.tensor(obs_full[:, :n].reshape(-1, D))
    if ref['zf'] is not None:
        x = ref['zf'].forward(x)
    with torch.no_grad():
        pdo = onets.ppo_actor(x.double(), [(w_.double(), b_.double()) for w_, b_ in ref['layers']],
                              ref['log_var'].double()).numpy().reshape(K, n, 2 * A)
    pdo[:, :, A:] *= np.exp(ref['noise'])[actors, None, None]
    worst['pd'] = max(worst['pd'], _ratio(pd, pdo))
    stats['mean_max'] = max(stats['mean_max'], float(np.abs(pdo[:, :, :A]).max()))
    # (b) actions for the known draws on the oracle's pd rows
    worst['act'] = max(worst['act'], _ratio(act, np.clip(eps * pdo[:, :, A:] + pdo[:, :, :A], -1, 1), absolute=True))
    # (c) env dynamics on what was staged, every step of every window
    nxt, r_or = philox.synth_env_step(obs_full[:, :n].reshape(-1, D), act.reshape(-1, A), ref['Ws'], ref['Wa'],
                                      env.seed + 7, steps.reshape(-1, 1), np.repeat(actors, n))
    worst['obs'] = max(worst['obs'], _ratio(obs_full[:, 1:].reshape(-1, D), nxt))
    worst['rew'] = max(worst['rew'], _ratio(rew.reshape(-1), r_or))
    # ... and the first observation of a window that opens an episode is the reset state
    for k in range(K):
        t0, i = int(steps[k, 0]), int(actors[k])
        if t0 not in _episode_starts(c, i):
            continue
        if t0 == 0:
            np.testing.assert_array_equal(obs_full[k, 0], ref['s0'][i])
        else:
            _, _, rz = philox.env_noise(env.seed + 7, t0 - 1, [i], D)
            worst['obs'] = max(worst['obs'], _ratio(obs_full[k, 0], rz[0]))
        stats['resets'] += 1


def _check_run(c, driver, ag, w, env, R, ref):
    """Everything the run left behind against the oracle.  -> the discrete state, for the cross-path comparison."""
    events = _oracle_events(c)
    q = OFIFO(c.mem, c.N)
    for e in events:
        q.insert(e)
    st = R._read_state()
    assert st['count'] == len(q) and st['total_in'] == len(events) and st['dropped'] == len(events) - len(q), \
        (st, len(q), len(events))
    assert st['capacity'] == c.mem + 3 and st['total_out'] == 0
    assert int(env.step_counter.item()) == c.T
    pos, ep = _oracle_actor_state(c)
    np.testing.assert_array_equal(w.stage_pos.cpu().numpy(), pos)
    np.testing.assert_array_equal(env.ep_step.cpu().numpy(), ep)
    expect = list(q.q)
    worst = dict(pd=0.0, act=0.0, obs=0.0, rew=0.0)
    stats = dict(clipped=0, records=0, resets=0, mean_max=0.0)
    dones = []
    at = 0
    while at < len(expect):
        k = min(len(expect) - at, c.mem, 1024)
        b = R.sample(k)
        _check_batch(c, ag, env, ref, expect[at:at + k], b, worst, stats)
        dones.append(b['dones'].cpu().numpy())
        at += k
    assert len(R) == 0 and stats['records'] == len(expect) > 0
    for k_, v in worst.items():
        assert v <= 1.0, '%s[%s] %s: error / bar = %.3f' % (c.name, driver, k_, v)
    assert stats['mean_max'] > 0.1                        # a live, non-trivial policy head
    assert stats['clipped'] > 0                           # the clip is exercised
    assert stats['resets'] > 0 or c.L == 0 or c.T < c.L
    print('%s[%s] records %d, resets %d, worst err/bar: %s' % (c.name, driver, stats['records'], stats['resets'],
                                                               ', '.join('%s %.3f' % kv for kv in worst.items())))
    return dict(state=st, ctr=int(env.step_counter.item()), pos=w.stage_pos.cpu().numpy(),
                ep=env.ep_step.cpu().numpy(), dones=np.concatenate(dones))


def _check_both_paths(c):
    """Case ``c`` on the persistent kernel (where its plan fits) and on the per-step launch path: both against the
    oracle, and the two against each other on every discrete quantity."""
    out = []
    for driver in (['chunk', 'step'] if c.supported else ['step']):
        out.append(_check_run(c, driver, *_drive(c, driver)))
    if len(out) == 2:
        p, s = out
        assert p['state'] == s['state'] and p['ctr'] == s['ctr']
        for k in ['pos', 'ep', 'dones']:
            np.testing.assert_array_equal(p[k], s[k], err_msg=k)


@pytest.mark.parametrize('ep_len,chunks', [(200, 3), (128, 2)])
def test_persistent_rollout_matches_oracle_at_cfg2_shape(ep_len, chunks):
    """BASELINE configs[1]: 1024 lockstep actors, n == stride == chunk == 128, episodes of 200 and 128 steps."""
    _check_both_paths(Case('cfg1_ep%d' % ep_len, (64, 256, 256, 8), 1024, 128, 128, 4 * 1024, ep_len, [128] * chunks,
                           stagger=False))


@pytest.mark.parametrize('name', list(CASES))
def test_rollout_matches_oracle(name):
    """The kernel's shape envelope and config edges, staggered episodes (see CASES)."""
    _check_both_paths(CASES[name])


def test_rollout_graph_replay_matches_oracle():
    """agent.main_loop as production drives it: the chunk is captured into a CUDA graph once and replayed.  Every
    replay must read the device step counter afresh and carry stage_pos / ep_step over from the previous chunk."""
    c = Case('graph', (64, 256, 256, 8), 256, 8, 5, 2000, 20, [13, 13, 13])
    _check_run(c, 'graph', *_drive(c, 'graph'))

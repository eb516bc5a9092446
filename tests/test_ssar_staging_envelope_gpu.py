"""The actor side of the off-policy algorithms against plain restatements, across its envelope.

n-step SSAR staging (sb200_ssar_step_f32 / sb200_ssar_step_host_f32: ssar_flags_kernel, ssar_commit_kernel), driven
through ExpSenderWrapperSSARNStepBootstrap into a UniformReplay, against oracle.windowing.SsarBatch -- the batched model
pinned to the reference's wrapper by tests/test_windowing_ref.py.  After EVERY step, bit for bit: the whole ring (slots
never written included), the ring's control block, the step counter, and every actor's pending deque with its float64
reward sums.  Observations and actions are float32 bit patterns that encode (actor, step, component), so a record
copied from the wrong actor, step or column cannot pass.  Device envs give float32 rewards; host envs give float64
rewards that float32 cannot hold, and a reset observation different from the successor.

DDPG exploration on the Philox path (unit_noise = NULL): sb200_ddpg_noise_f32's draws against oracle.philox.agent_eps,
its output against the float64 formula, and sb200_ddpg_ou_noise_f32's float64 state against numpy's recurrence.  Every
bar quotes the worst value measured on an H100 80GB HBM3 next to it."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import ddpg_configs
from oracle.philox import agent_eps
from oracle.windowing import SsarBatch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32 = np.float32
ACT = np.uint32(1 << 31)


def _lib_():
    from surreal_b200 import _lib, ops
    ops._stream()
    return _lib.lib()


def _st():
    from surreal_b200 import ops
    return ops._stream()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


# ------------------------------------------------------------------------------------------------------------------
# A. n-step SSAR staging
def _obs_code(i, t, reset):
    """float32 bit pattern of component 0 of actor i's observation after its t-th step; component d adds d."""
    return (np.asarray(i, np.uint32) << np.uint32(19)) | np.uint32(t << 10) | np.uint32(512 if reset else 0)


def _act_code(i, t):
    return ACT | (np.asarray(i, np.uint32) << np.uint32(19)) | np.uint32(t << 10)


def _rows(codes, width):
    return (np.asarray(codes, np.uint32)[..., None] + np.arange(width, dtype=np.uint32)).view(F32)


class Script:
    """N actors over T steps: episode lengths per actor (cycled), done flags, rewards, and the payload codes."""

    def __init__(self, N, T, scripts, rew64, seed):
        assert T < 511 and N < 4080
        rng = np.random.default_rng(seed)
        self.N, self.T = N, T
        self.done = np.zeros((T, N), F32)
        for i, s in enumerate(scripts):
            t, k = 0, 0
            while True:
                t += s[k % len(s)]
                k += 1
                if t > T:
                    break
                self.done[t - 1, i] = 1.0
        r = rng.standard_normal((T, N)) * 3.0
        self.rew = r if rew64 else r.astype(F32)
        if rew64:
            assert np.all(r.astype(F32).astype(np.float64) != r)
        ids = np.arange(N)
        self.obs0 = _obs_code(ids, 0, True)
        self.nxt = [_obs_code(ids, t + 1, False) for t in range(T)]
        self.reset = [np.where(self.done[t] > 0, _obs_code(ids, t + 1, True), self.nxt[t]) for t in range(T)]
        self.act = [_act_code(ids, t) for t in range(T)]


class DeviceEnv:
    def __init__(self, s, D, A):
        self.s, self.N, self.D, self.A, self.t = s, s.N, D, A, 0
        self.device = torch.device(DEV)

    def _dev(self, codes):
        return torch.from_numpy(_rows(codes, self.D).copy()).to(DEV)

    def reset(self):
        self.t = 0
        return {'low_dim': {'flat_inputs': self._dev(self.s.obs0)}}, {}

    def step(self, action):
        s, t = self.s, self.t
        self.t += 1
        return ({'low_dim': {'flat_inputs': self._dev(s.reset[t])}}, torch.from_numpy(s.rew[t].copy()).to(DEV),
                torch.from_numpy(s.done[t].copy()).to(DEV), {'obs_next': self._dev(s.nxt[t])})


class HostEnv:
    def __init__(self, s, D, A):
        self.s, self.N, self.D, self.A, self.t = s, s.N, D, A, 0

    def reset(self):
        self.t = 0
        return {'low_dim': {'flat_inputs': _rows(self.s.obs0, self.D)}}, {}

    def step(self, action):
        s, t = self.s, self.t
        self.t += 1
        return ({'low_dim': {'flat_inputs': _rows(s.reset[t], self.D)}}, s.rew[t].copy(), s.done[t].copy(),
                {'obs_next': _rows(s.nxt[t], self.D)})


def _scripts(N, n, kind):
    if kind == 'unstaggered':                  # every actor emits at the same steps: K = N records in one step
        return [[n + 3]] * N
    base = [1, max(n - 1, 1), n, 2 * n + 1, 3, 1, n + 4, 7]
    return [base[i % len(base):] + base[:i % len(base)] for i in range(N)]


# (N, n_step, D, A, capacity, gamma, episodes, host env, T)
CASES = {
    'one_actor_cap1':     (1, 3, 1, 1, 1, 0.99, 'staggered', False, 40),
    'one_actor_host':     (1, 5, 3, 3, 1000, 0.37, 'staggered', True, 40),
    'dqn_shape':          (31, 1, 131, 1, 17, 0.99, 'staggered', False, 30),
    'n2_wide_host':       (31, 2, 300, 130, 97, 0.0, 'staggered', True, 24),
    'n16_gamma1':         (31, 16, 131, 3, 4099, 1.0, 'staggered', False, 60),
    'chunk_1024_k_gt_cap': (1024, 3, 3, 3, 509, 0.99, 'unstaggered', False, 30),
    'chunk_1024_host':    (1024, 5, 1, 3, 4099, 0.37, 'staggered', True, 40),
    'chunk_1025':         (1025, 3, 1, 1, 4099, 0.99, 'staggered', False, 40),
    'chunk_1025_k_gt_cap_host': (1025, 2, 2, 1, 1021, 0.99, 'unstaggered', True, 20),
    'three_chunks':       (2500, 3, 2, 3, 131071, 0.99, 'staggered', False, 40),
    'three_chunks_host':  (2500, 16, 1, 1, 7919, 0.37, 'staggered', True, 40),
    'three_chunks_gamma0_cap1': (2500, 5, 1, 1, 1, 0.0, 'unstaggered', False, 20),
}


def _wrapper(N, n, D, A, cap, gamma, host, s):
    from surreal_b200.replay import UniformReplay
    from surreal_b200.env import ExpSenderWrapperSSARNStepBootstrap as W
    lc, ec, sc = ddpg_configs(D=D, A=A, n_step=n, memory_size=cap, start=0)
    lc.algo.gamma = gamma
    R = UniformReplay(lc, ec, sc)
    env = (HostEnv if host else DeviceEnv)(s, D, A)
    w = W(env, lc, sc, replay=R)
    assert w.host_env == host
    return w, R


class Expected:
    """The ring as the oracle's Uniform holds it, as float32 bit patterns; unwritten slots are zero."""

    def __init__(self, m, D, A):
        self.m, self.D, self.A = m, D, A
        cap = m.ring.memory_size
        self.written = np.zeros(cap, bool)
        self.obs = np.zeros(cap, np.uint32)
        self.nxt = np.zeros(cap, np.uint32)
        self.act = np.zeros(cap, np.uint32)
        self.rew = np.zeros(cap, F32)
        self.done = np.zeros(cap, F32)
        self.seen = 0

    def update(self):
        m, cap = self.m, self.m.ring.memory_size
        for k in range(self.seen, m.total_in):
            o, on, a, r, d = m.ring.mem[k % cap]
            s = k % cap
            self.written[s] = True
            self.obs[s], self.nxt[s], self.act[s], self.rew[s], self.done[s] = o, on, a, F32(r), float(d)
        self.seen = m.total_in

    def rows(self, codes, width):
        out = _rows(codes, width).view(np.uint32)
        out[~self.written] = 0
        return out


def _u32(t):
    return t.cpu().numpy().view(np.uint32)


def _compare(w, R, m, ex, n, D, A, step):
    """-> {field: mismatching elements} after ``step`` steps."""
    bad = {}
    ex.update()
    bad['r_obs'] = int((_u32(R.r_obs) != ex.rows(ex.obs, D)).sum())
    bad['r_obs_next'] = int((_u32(R.r_obs_next) != ex.rows(ex.nxt, D)).sum())
    bad['r_act'] = int((_u32(R.r_act) != ex.rows(ex.act, A)).sum())
    bad['r_rew'] = int((_u32(R.r_rew) != ex.rew.view(np.uint32)).sum())
    bad['r_done'] = int((_u32(R.r_done) != ex.done.view(np.uint32)).sum())
    bad['state'] = int((R.state.cpu().numpy() != np.array(m.state())).sum())
    bad['step_counter'] = int(int(w.step_counter.item()) != step)
    N = m.N
    lens = np.array([len(m.last_n[i]) for i in range(N)])
    got_len = w.dq_len.cpu().numpy()
    bad['dq_len'] = int((got_len != lens).sum())
    mask = np.arange(n)[None, :] < lens[:, None]
    e_obs = np.zeros((N, n), np.uint32)
    e_act = np.zeros((N, n), np.uint32)
    e_sum = np.zeros((N, n), np.float64)
    for i in range(N):
        for k, (o, a, r) in enumerate(m.pending(i)):
            e_obs[i, k], e_act[i, k], e_sum[i, k] = o, a, r
    bad['dq_obs'] = int((_u32(w.dq_obs)[mask] != _rows(e_obs, D).view(np.uint32)[mask]).sum())
    bad['dq_act'] = int((_u32(w.dq_act)[mask] != _rows(e_act, A).view(np.uint32)[mask]).sum())
    bad['dq_rew'] = int((w.dq_rew.cpu().numpy().view(np.uint64)[mask] != e_sum.view(np.uint64)[mask]).sum())
    return bad


def _assert_clean(report, tag):
    failing = {k: v for k, v in report['total'].items() if v}
    assert not failing, '%s: mismatching elements %s, first at step %s' % (tag, failing, report['first'])


def _record(report, bad, step):
    for k, v in bad.items():
        report['total'][k] = report['total'].get(k, 0) + v
        if v and k not in report['first']:
            report['first'][k] = step


def _snapshot(w, R):
    return [t.clone() for t in (w.dq_len, w.dq_obs, w.dq_act, w.dq_rew, w._obs, R.r_obs, R.r_obs_next, R.r_act,
                                R.r_rew, R.r_done, R.state, w.step_counter)]


def _restore(w, R, snap):
    for t, v in zip((w.dq_len, w.dq_obs, w.dq_act, w.dq_rew, w._obs, R.r_obs, R.r_obs_next, R.r_act, R.r_rew,
                     R.r_done, R.state, w.step_counter), snap):
        t.copy_(v)


def _graph_replay(w, R, s, D, A, t0, steps, eager):
    """Steps t0 .. t0 + steps - 1 again from the snapshot taken before t0: one captured sb200_ssar_step_f32 on fixed
    input buffers, refilled before each replay.  Must give the eager run's bits."""
    L = _lib_()
    o_b = torch.empty_like(w._obs)
    a_b = torch.empty(s.N, A, device=DEV)
    on_b = torch.empty(s.N, D, device=DEV)
    r_b = torch.empty(s.N, device=DEV)
    d_b = torch.empty(s.N, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        rc = L.sb200_ssar_step_f32(C.byref(w.ssar), _p(o_b), _p(a_b), _p(on_b), _p(r_b), _p(d_b), _st())
    assert rc == 0
    torch.cuda.synchronize()
    o_b.copy_(w._obs)
    for t in range(t0, t0 + steps):
        a_b.copy_(torch.from_numpy(_rows(s.act[t], A).copy()))
        on_b.copy_(torch.from_numpy(_rows(s.nxt[t], D).copy()))
        r_b.copy_(torch.from_numpy(s.rew[t].copy()))
        d_b.copy_(torch.from_numpy(s.done[t].copy()))
        g.replay()
        o_b.copy_(torch.from_numpy(_rows(s.reset[t], D).copy()))
    torch.cuda.synchronize()
    got = _snapshot(w, R)
    names = ('dq_len', 'dq_obs', 'dq_act', 'dq_rew', 'obs', 'r_obs', 'r_obs_next', 'r_act', 'r_rew', 'r_done', 'state',
             'step_counter')
    for name, a, b in zip(names, got, eager):
        if name == 'obs':
            continue                                      # the graph's s_t lives in o_b
        # dq_* beyond each deque's length hold stale entries that only the next steps may touch: compare it all anyway,
        # the graph launches the same kernels on the same bytes
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), name


@pytest.mark.parametrize('case', list(CASES))
def test_ssar_staging_envelope_matches_batched_reference_model(case):
    N, n, D, A, cap, gamma, kind, host, T = CASES[case]
    s = Script(N, T, _scripts(N, n, kind), rew64=host, seed=list(CASES).index(case))
    w, R = _wrapper(N, n, D, A, cap, gamma, host, s)
    m = SsarBatch(N, n, gamma, cap)
    ex = Expected(m, D, A)
    w.reset()
    m.reset(list(s.obs0))
    report = {'total': {}, 'first': {}}
    t_graph, g_steps, snap = T // 2, 3, None
    emitted_max = 0
    for t in range(T):
        if not host and t == t_graph:
            torch.cuda.synchronize()
            snap = _snapshot(w, R)
        a = torch.from_numpy(_rows(s.act[t], A).copy())
        w.step(a.numpy() if host else a.to(DEV))
        before = m.total_in
        m.step(list(s.act[t]), list(s.nxt[t]), list(s.rew[t]), list(s.done[t] > 0), obs_reset=list(s.reset[t]))
        emitted_max = max(emitted_max, m.total_in - before)
        torch.cuda.synchronize()
        _record(report, _compare(w, R, m, ex, n, D, A, t + 1), t + 1)
        if not host and t == t_graph + g_steps - 1:
            eager = _snapshot(w, R)
    _assert_clean(report, case)
    assert m.total_in > 0
    if kind == 'unstaggered' and cap < N:
        assert emitted_max > cap                         # the K > capacity drop rule was exercised
    if not host:
        cur = _snapshot(w, R)
        _restore(w, R, snap)
        _graph_replay(w, R, s, D, A, t_graph, g_steps, eager)
        _restore(w, R, cur)


def test_ssar_staging_accepts_n_step_64_and_refuses_65():
    """n_step = 64, the cap of the gamma^k table, stages as the model does; 65 is refused before any launch: the step
    raises and neither the ring, its control block, the deques nor the step counter change."""
    from surreal_b200._lib import SB200Error
    N, D, A, T = 3, 2, 1, 70
    s = Script(N, T, [[T + 1], [66], [1, 64]], rew64=False, seed=5)
    w, R = _wrapper(N, 64, D, A, 128, 0.99, False, s)
    m = SsarBatch(N, 64, 0.99, 128)
    ex = Expected(m, D, A)
    w.reset()
    m.reset(list(s.obs0))
    report = {'total': {}, 'first': {}}
    for t in range(T):
        w.step(torch.from_numpy(_rows(s.act[t], A).copy()).to(DEV))
        m.step(list(s.act[t]), list(s.nxt[t]), list(s.rew[t]), list(s.done[t] > 0), obs_reset=list(s.reset[t]))
        torch.cuda.synchronize()
        _record(report, _compare(w, R, m, ex, 64, D, A, t + 1), t + 1)
    _assert_clean(report, 'n_step 64')
    assert m.total_in > 0

    w2, R2 = _wrapper(N, 65, D, A, 128, 0.99, False, s)
    w2.reset()
    R2.r_obs.fill_(7.0)
    before = _snapshot(w2, R2)
    with pytest.raises(SB200Error, match='sb200_ssar_step_f32'):
        w2.step(torch.from_numpy(_rows(s.act[0], A).copy()).to(DEV))
    torch.cuda.synchronize()
    for a, b in zip(_snapshot(w2, R2), before):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------------
# B. DDPG exploration noise on the Philox path
NOISE_ULP_BAR = 8
SEED = 0x5EED


def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(F32)).astype(np.float64)


def _noise(L, mean, sigma, N, A, ctr, det=0, unit=None):
    """sb200_ddpg_noise_f32 on a [N, ldm] mean with NaN past column A; -> action [N, A]."""
    ldm = mean.shape[1]
    m = torch.from_numpy(np.ascontiguousarray(mean, F32)).to(DEV)
    sg = torch.from_numpy(np.ascontiguousarray(sigma, F32)).to(DEV)
    c = torch.tensor([ctr], dtype=torch.int64, device=DEV)
    out = torch.full((N, A), float('nan'), device=DEV)
    rc = L.sb200_ddpg_noise_f32(_p(m), ldm, _p(sg), _p(unit), N, A, det, C.c_uint64(SEED), _p(c), _p(out), _st())
    assert rc == 0
    torch.cuda.synchronize()
    assert int(c.item()) == ctr                           # the noise kernel reads the counter, it does not advance it
    return out.cpu().numpy()


def _padded_mean(vals, ldm):
    out = np.full((vals.shape[0], ldm), np.nan, F32)
    out[:, :vals.shape[1]] = vals
    return out


def _draws(L, N, A, ctr):
    """The kernel's own N(0,1) draws: mean 0, sigma 2^-3, |e| < 6.7, so the output times 8 is e exactly."""
    return _noise(L, np.zeros((N, A + 3), F32), np.full(N, 0.125, F32), N, A, ctr) * F32(8)


def _noise_ref(mean, sigma, e):
    """clip(float32(double(clip(mean)) + double(sigma) * double(e))), in float64."""
    m = np.clip(mean.astype(F32), -1, 1).astype(np.float64)
    a = (m + sigma.astype(F32).astype(np.float64)[:, None] * e.astype(F32).astype(np.float64)).astype(F32)
    return np.clip(a, F32(-1), F32(1))


@pytest.mark.parametrize('A', [1, 3, 4, 5, 17])
@pytest.mark.parametrize('N', [1, 255, 256, 257, 5000])
def test_ddpg_noise_philox_draws_and_outputs(N, A):
    """unit_noise = NULL: the draws are action_noise4 keyed (seed, *step_counter, actor << 16 | quad).  Read back
    exactly, against oracle.philox.agent_eps (float64 libm) within NOISE_ULP_BAR; measured worst 3.  Live means beyond
    +-1, per-actor sigma (some 0), ldm > A: with the kernel's draws the output is the float64 formula bit for bit; with
    the oracle's, within the bar in ulp of max(|out|, |sigma e|); measured worst 3.  Deterministic: clip(mean)."""
    L = _lib_()
    rng = np.random.default_rng(N * 31 + A)
    worst = worst2 = 0.0
    ldm = A + 3
    for ctr in (0, 7, (1 << 40) + 3):
        e_ref = agent_eps(SEED, ctr, np.arange(N), A)
        e = _draws(L, N, A, ctr)
        u = float((np.abs(e.astype(np.float64) - e_ref) / _ulp(e_ref)).max())
        worst = max(worst, u)
        assert u <= NOISE_ULP_BAR, (ctr, u)
        mean = (rng.standard_normal((N, A)) * 1.5).astype(F32)
        mean[0, 0] = 3.0
        mean[-1, -1] = -2.5
        sigma = rng.uniform(0.0, 0.6, N).astype(F32)
        sigma[::3] = 0.0
        got = _noise(L, _padded_mean(mean, ldm), sigma, N, A, ctr)
        np.testing.assert_array_equal(got.view(np.uint32), _noise_ref(mean, sigma, e).view(np.uint32))
        want = _noise_ref(mean, sigma, e_ref)
        scale = np.maximum(np.abs(want).astype(np.float64), np.abs(sigma[:, None] * e_ref.astype(np.float64)))
        u2 = float((np.abs(got.astype(np.float64) - want) / _ulp(np.maximum(scale, 2.0 ** -20))).max())
        worst2 = max(worst2, u2)
        assert u2 <= NOISE_ULP_BAR, (ctr, u2)
        det = _noise(L, _padded_mean(mean, ldm), sigma, N, A, ctr, det=1)
        np.testing.assert_array_equal(det, np.clip(mean, F32(-1), F32(1)))
    if N > 1:
        assert not np.array_equal(e[0], e[1])           # actors draw from distinct streams
    print('measured ddpg_noise', N, A, 'draw ulp', worst, 'out ulp', worst2)


def _ou(L, mean, sigma64, state, N, A, ctr, theta, dt, det=0):
    ldm = mean.shape[1]
    m = torch.from_numpy(np.ascontiguousarray(mean, F32)).to(DEV)
    sg = torch.from_numpy(np.ascontiguousarray(sigma64, np.float64)).to(DEV)
    c = torch.tensor([ctr], dtype=torch.int64, device=DEV)
    out = torch.full((N, A), float('nan'), device=DEV)
    rc = L.sb200_ddpg_ou_noise_f32(_p(m), ldm, _p(sg), C.c_void_p(0), N, A, det, C.c_uint64(SEED), _p(c), theta, dt,
                                   _p(state), _p(out), _st())
    assert rc == 0
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize('N,A', [(1, 1), (257, 3), (5000, 5), (40, 17)])
def test_ddpg_ou_noise_state_is_numpys_recurrence(N, A):
    """Eight OU steps with per-actor float64 sigma, counters c, c+1, ...: the draws are the Gaussian kernel's at the same
    (seed, counter); the float64 state equals numpy's left-to-right x + theta*(0 - x)*dt + sigma*sqrt(dt)*e bit for
    bit, and the action clip(float32(double(clip(mean)) + x)) too.  Deterministic mode leaves the state untouched."""
    L = _lib_()
    rng = np.random.default_rng(N + A)
    theta, dt = 0.15, 1e-2
    sigma = rng.uniform(0.05, 0.4, N)
    sigma[0] = 0.3 + 1e-12                                # not a float32 value
    x = np.zeros((N, A))
    state = torch.zeros(N, A, dtype=torch.float64, device=DEV)
    ctr0 = (1 << 40) + 3
    for k in range(8):
        ctr = ctr0 + k
        e = _draws(L, N, A, ctr).astype(np.float64)
        mean = (rng.standard_normal((N, A)) * 1.5).astype(F32)
        got = _ou(L, _padded_mean(mean, A + 2), sigma, state, N, A, ctr, theta, dt)
        x = x + theta * (0.0 - x) * dt + sigma[:, None] * np.sqrt(dt) * e
        np.testing.assert_array_equal(state.cpu().numpy().view(np.uint64), x.view(np.uint64))
        want = np.clip((np.clip(mean, F32(-1), F32(1)).astype(np.float64) + x).astype(F32), F32(-1), F32(1))
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    before = state.clone()
    mean = (rng.standard_normal((N, A)) * 1.5).astype(F32)
    det = _ou(L, _padded_mean(mean, A + 2), sigma, state, N, A, ctr0 + 8, theta, dt, det=1)
    assert torch.equal(state, before)
    np.testing.assert_array_equal(det, np.clip(mean, F32(-1), F32(1)))

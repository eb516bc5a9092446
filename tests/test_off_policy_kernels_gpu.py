"""The off-policy update kernels against plain float32 / float64 restatements at their edges: the Bellman targets of DDPG
and TD3 with their statistics and bad-action flag, TD3's target-policy smoothing with injected and Philox draws, the soft
and hard target updates, the weighted (prioritized-replay) DDPG update against float64 autograd, and a bad record first
drawn in the middle of a K-update call.  The kernels are called through the C ABI; every bar quotes the worst value
measured on an H100 80GB HBM3 next to it."""
import ctypes as C

import numpy as np
import pytest
import torch

import grad_ref as R
from helpers import ddpg_configs
from oracle.philox import agent_eps
from test_ddpg_device_engine_gpu import _replay, _set_view
from test_dqn_gpu import _filled_replay, dqn_configs
from test_grads_gpu import _check_grads, _dev, _layers
from test_prioritized_replay_gpu import _fill_ring, _per
from test_uniform_device_sampler import device_sample_indices

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NAN, INF = float('nan'), float('inf')
F32 = np.float32
DS = dict(ACTOR_LOSS=0, CRITIC_LOSS=1, ACTION_NORM=2, REWARDS=3, Q_TARGET=4, Q_POLICY=5, ABSMAX=6, TD_ERROR=7,
          IS_WEIGHT=8)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _lib_():
    from surreal_b200 import _lib, ops
    ops._stream()                     # sb200_init once
    return _lib.lib()


def _st():
    from surreal_b200 import ops
    return ops._stream()


def _check(rc, what):
    from surreal_b200 import _lib
    _lib.check(rc, what)


def _padded(vals, ld):
    """[rows, ld] device buffer holding ``vals`` (numpy [rows, w]) in its first columns, NaN sentinels after them."""
    out = torch.full((vals.shape[0], ld), NAN, device=DEV)
    out[:, :vals.shape[1]] = torch.from_numpy(np.ascontiguousarray(vals, dtype=F32)).to(DEV)
    return out


def _ulp(x):
    """float64 array of the fp32 ulp at |x|."""
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(F32)).astype(np.float64)


# ------------------------------------------------------------------------------------------------------------------
# A. Bellman target kernels
GAMMA = 0.99


def _target_case(B, A, seed):
    rng = np.random.default_rng(seed)
    r = (rng.standard_normal(B) * 2).astype(F32)
    q = (rng.standard_normal(B) * 10).astype(F32)
    q2 = (rng.standard_normal(B) * 10).astype(F32)
    d = (rng.random(B) < 0.3).astype(F32)
    d[:min(B, 2)] = (0.0, 1.0)[:min(B, 2)]
    a = rng.uniform(-1, 1, (B, A)).astype(F32)
    a[::7, 0] = 1.0                                       # |a| == 1 exactly is in range
    a[3::11, A - 1] = -1.0
    return r, q, q2, d, a


def _run_target(L, ws, bufs, B, A, disc, two, lda, stats=None):
    r_d, q_d, q2_d, d_d, a_d = bufs
    y = torch.full((B,), NAN, device=DEV)
    stats = torch.full((16,), NAN, device=DEV) if stats is None else stats
    if two:
        _check(L.sb200_ddpg_target2_f32(_p(r_d), _p(q_d), q_d.stride(0), _p(q2_d), q2_d.stride(0), _p(d_d), _p(a_d), lda,
                                        B, A, disc, _p(y), _p(stats), _p(ws), _st()), 'target2')
    else:
        _check(L.sb200_ddpg_target_f32(_p(r_d), _p(q_d), q_d.stride(0), _p(d_d), _p(a_d), lda, B, A, disc, _p(y),
                                       _p(stats), _p(ws), _st()), 'target')
    torch.cuda.synchronize()
    return y.cpu().numpy(), stats.cpu().numpy()


def _bad_flag(L, ws):
    off = int(L.sb200_ddpg_bad_action_offset())
    return int(ws[off:off + 4].view(torch.int32).item())


def _target_bufs(r, q, q2, d, a, lda):
    return (torch.from_numpy(r).to(DEV), _padded(q[:, None], 2), _padded(q2[:, None], 3), torch.from_numpy(d).to(DEV),
            _padded(a, lda))


Y_ULP_BAR, STAT_BAR = 2.0, 3e-7


@pytest.mark.parametrize('A', [1, 3, 8, 17])
@pytest.mark.parametrize('B', [1, 255, 256, 257, 4096, 65537])
def test_bellman_target_kernels_against_float32_and_float64(B, A):
    """y bit-exact against r + (float32(gamma^n) q') (1 - done) in numpy float32 (the reference's operation order), and
    min(y, y2) for TD3.  Against float64, in ulp of the largest of |r|, |gamma^n q' (1 - done)| and |y| (a cancelling
    sum has no error bound in ulp of y itself): measured worst 1.16, bar Y_ULP_BAR = 2 (three roundings, one of them
    float32(gamma^n)).  Statistics against float64 sums over the whole batch, error / max(1, |v|): measured worst
    6.5e-8, bar STAT_BAR = 3e-7; the absmax is exact.  A second call on the same workspace returns the same bits: the
    last-block ticket reset itself."""
    L = _lib_()
    lda = A + 3
    r, q, q2, d, a = _target_case(B, A, B * 31 + A)
    bufs = _target_bufs(r, q, q2, d, a, lda)
    ws = torch.zeros(int(L.sb200_ddpg_workspace_bytes(B)), dtype=torch.uint8, device=DEV)
    worst_u = worst_s = 0.0
    for n in (1, 3):
        disc = float(pow(GAMMA, n))
        t32 = (F32(disc) * q) * (F32(1) - d)
        t32_2 = (F32(disc) * q2) * (F32(1) - d)
        y32 = r + t32
        t64 = disc * q.astype(np.float64) * (1.0 - d.astype(np.float64))
        y64 = r.astype(np.float64) + t64
        for two in (False, True):
            want = np.minimum(y32, r + t32_2) if two else y32
            w64 = np.minimum(y64, r + disc * q2.astype(np.float64) * (1.0 - d)) if two else y64
            got = [_run_target(L, ws, bufs, B, A, disc, two, lda) for _ in range(2)]
            assert np.array_equal(got[0][0], got[1][0]) and np.array_equal(got[0][1], got[1][1], equal_nan=True)
            assert _bad_flag(L, ws) == 0
            y, s = got[0]
            assert np.array_equal(y.view(np.int32), want.view(np.int32)), ('y', n, two)
            tt = np.where(w64 == y64, np.abs(t64), np.abs(disc * q2.astype(np.float64) * (1.0 - d)))
            scale = _ulp(np.maximum(np.maximum(np.abs(r), tt), np.abs(w64)))
            u = float((np.abs(y.astype(np.float64) - w64) / scale).max())
            worst_u = max(worst_u, u)
            assert u <= Y_ULP_BAR, ('y vs float64', n, two, u)
            a64 = a.astype(np.float64)
            exp = {'REWARDS': r.astype(np.float64).mean(), 'ACTION_NORM': np.sqrt((a64 ** 2).sum(1)).mean(),
                   'Q_TARGET': w64.mean()}
            for k, v in exp.items():
                e = abs(float(s[DS[k]]) - v) / max(1.0, abs(v))
                worst_s = max(worst_s, e)
                assert e <= STAT_BAR, (k, n, two, float(s[DS[k]]), v)
            assert s[DS['ABSMAX']] == np.abs(a).max()
            assert np.isnan(s[DS['ACTOR_LOSS']]) and np.isnan(s[DS['Q_POLICY']])   # nothing else written
    print('measured target', B, A, 'y ulp', worst_u, 'stats', worst_s)


BAD_VALUES = [float(np.nextafter(F32(1), F32(2))), float(np.nextafter(F32(-1), F32(-2))), INF, -INF, NAN]


@pytest.mark.parametrize('two', [False, True])
@pytest.mark.parametrize('B,row', [(4096, 5), (257, 256)])
def test_bad_action_flag_edges(B, row, two):
    """The flag is 0 for |a| == 1 exactly and 1 for the next float32 beyond either bound, for +-inf and for NaN (the
    reference's `actions.max() <= 1` propagates NaN, so it rejects one); the bad row sits in block 0 (4096, row 5) or
    alone in the last, partial block (257, row 256).  A following good call clears the flag."""
    L = _lib_()
    A, lda = 3, 5
    r, q, q2, d, a = _target_case(B, A, 7)
    a[:, 1] = 1.0
    a[1::2, 1] = -1.0
    ws = torch.zeros(int(L.sb200_ddpg_workspace_bytes(B)), dtype=torch.uint8, device=DEV)
    good = _target_bufs(r, q, q2, d, a, lda)
    _, s = _run_target(L, ws, good, B, A, GAMMA, two, lda)
    assert _bad_flag(L, ws) == 0 and s[DS['ABSMAX']] == 1.0
    for v in BAD_VALUES:
        ab = a.copy()
        ab[row, 2] = v
        y, s = _run_target(L, ws, _target_bufs(r, q, q2, d, ab, lda), B, A, GAMMA, two, lda)
        assert _bad_flag(L, ws) == 1, ('bad action not flagged', v, B, row)
        assert not (s[DS['ABSMAX']] <= 1.0), ('absmax', v, s[DS['ABSMAX']])
        _run_target(L, ws, good, B, A, GAMMA, two, lda)
        assert _bad_flag(L, ws) == 0, ('flag not cleared after', v)


# ------------------------------------------------------------------------------------------------------------------
# B. TD3 target-policy smoothing
PN, NC = 0.2, 0.5


def _smooth_ref(pi, e, pn=PN, nc=NC):
    """The kernel's float32 restatement: clamp(pi + clip(float32(e) * float32(0.2), -0.5, 0.5), -1, 1)."""
    nz = np.minimum(np.maximum(e.astype(F32) * F32(pn), -F32(nc)), F32(nc))
    return np.minimum(np.maximum(pi.astype(F32) + nz, F32(-1)), F32(1))


def _smooth(L, pi, B, A, noise=None, seed=0, ctr=None, pn=PN, nc=NC):
    pi_d = _padded(pi, A + 2)
    out = torch.full((B, A + 1), NAN, device=DEV)
    e_d = torch.from_numpy(np.ascontiguousarray(noise, dtype=F32)).to(DEV) if noise is not None else None
    c_d = torch.tensor([ctr], dtype=torch.int64, device=DEV) if ctr is not None else None
    _check(L.sb200_ddpg_smooth_action_f32(_p(pi_d), A + 2, _p(e_d), B, A, pn, nc, seed, _p(c_d), _p(out), A + 1, _st()),
           'smooth')
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.isnan(o[:, A:]).all(), 'padding column written'
    return o[:, :A]


@pytest.mark.parametrize('B,A', [(1, 1), (255, 3), (257, 8), (4096, 17)])
def test_smoothing_with_injected_draws_is_bit_exact(B, A):
    """Injected N(0, 1) draws: bit-exact against the float32 restatement, including pi exactly +-1, noise exactly at
    +-clip (e = +-2.5: float32(2.5) * float32(0.2) rounds to 0.5), noise beyond it and sums past +-1."""
    L = _lib_()
    rng = np.random.default_rng(B + A)
    pi = np.tanh(rng.standard_normal((B, A)) * 2).astype(F32)
    e = rng.standard_normal((B, A)).astype(F32) * F32(2)
    pi[::3, 0] = 1.0
    pi[1::3, A - 1] = -1.0
    e[::5, 0] = 2.5
    e[2::5, A - 1] = -2.5
    e[4::9, 0] = -40.0
    assert F32(2.5) * F32(PN) == F32(NC)
    got = _smooth(L, pi, B, A, noise=e)
    want = _smooth_ref(pi, e)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    assert (np.abs(got) <= 1).all()
    if B > 2:
        assert (got == 1).any() and (got == -1).any()


SMOOTH_ULP_BAR = 8


@pytest.mark.parametrize('A', [1, 4, 5, 8])
@pytest.mark.parametrize('B', [1, 300, 4096])
def test_smoothing_philox_draws(B, A):
    """unit_noise = NULL: the draws are action_noise4 keyed (seed, *step_counter, row << 16 | quad), restated by
    oracle.philox.agent_eps with float64 log / sqrt / cos / sin; the device's are fp32.  Read back exactly with scale
    1/8 and no clip (|e| < 6.7 < 8, so out * 8 = e), they agree within measured worst 3 ulp, bar SMOOTH_ULP_BAR = 8.
    With the training constants (0.2, 0.5), out against the float32 restatement over the reference draws, in ulp of
    max(|out|, 0.5): measured worst 2, same bar."""
    L = _lib_()
    rng = np.random.default_rng(B * 3 + A)
    seed = 77
    worst = worst2 = 0.0
    for ctr in (0, 7, (1 << 40) + 3):
        e = agent_eps(seed, ctr, np.arange(B), A)
        raw = _smooth(L, np.zeros((B, A), F32), B, A, seed=seed, ctr=ctr, pn=0.125, nc=1e30) * F32(8)
        u = float((np.abs(raw.astype(np.float64) - e) / _ulp(e)).max())
        worst = max(worst, u)
        assert u <= SMOOTH_ULP_BAR, (ctr, u)
        pi = np.tanh(rng.standard_normal((B, A))).astype(F32)
        out = _smooth(L, pi, B, A, seed=seed, ctr=ctr)
        want = _smooth_ref(pi, e)
        u2 = float((np.abs(out.astype(np.float64) - want) / _ulp(np.maximum(np.abs(want), 0.5))).max())
        worst2 = max(worst2, u2)
        assert u2 <= SMOOTH_ULP_BAR, (ctr, u2)
    assert not np.array_equal(agent_eps(seed, 0, np.arange(B), A), agent_eps(seed, 7, np.arange(B), A))
    print('measured philox', B, A, 'draw ulp', worst, 'out ulp', worst2)


def test_td3_learner_consumes_one_counter_per_update():
    """learn_from_replay(K = 4) on a TD3 learner with Philox noise: the device counter advances by 4 per call and the
    last update smoothed its target actions with counter c + 3 (re-running the kernel on the saved target actions
    reproduces them bit for bit, and counter c does not).  A graph that replayed one draw K times would fail here."""
    from surreal_b200.learner import DDPGLearner
    r, _ = _replay(600, D=9, A=3, B=16, sampler_seed=3)
    _set_view(r, 590, 500)
    lc, ec, sc = ddpg_configs(D=9, A=3, B=16, target={'type': 'soft', 'tau': 0.05, 'interval': 1})
    lc.algo.network.use_double_critic = lc.algo.network.use_action_regularization = True
    torch.manual_seed(11)
    Lr = DDPGLearner(lc, ec, sc)
    Lr.use_cuda_graph = True
    L = _lib_()
    B, A = 16, 3
    for call in range(3):                                  # the later calls replay the captured graph
        c = int(Lr._td3_counter.item())
        Lr.learn_from_replay(r, updates=4)
        torch.cuda.synchronize()
        assert int(Lr._td3_counter.item()) == c + 4
        pi = Lr._pi_t.cpu().numpy()
        got = Lr._pi_t2.cpu().numpy()
        for k, same in ((3, True), (0, False)):
            again = _smooth(L, pi, B, A, seed=Lr._td3_seed, ctr=c + k)
            assert np.array_equal(again, got) == same, (call, k)


# ------------------------------------------------------------------------------------------------------------------
# C. target updates
SOFT_SIZES, SOFT_ULP_BAR = [1, 1023, 264 * 1024 + 5], 3.0


@pytest.mark.parametrize('n', SOFT_SIZES)
def test_soft_update(n):
    """t (1 - tau) + tau s: bit-exact against float32 with keep = float32(1) - float32(tau) (for the tau below that
    equals float32(1 - tau), the reference's scalar).  Against float64, in ulp of max(|t (1 - tau)|, |tau s|): measured
    worst 2.35 (tau 1e-3, n 270341), bar SOFT_ULP_BAR = 3.  Not 1: float32(1 - tau) alone is off by up to 2^-24
    relative, then come two products and a sum.  The last size runs the grid-stride loop (264 blocks).  A raised stop
    flag changes nothing."""
    L = _lib_()
    g = torch.Generator().manual_seed(n)
    t0 = torch.randn(n, generator=g)
    s = torch.randn(n, generator=g)
    s_d = s.to(DEV)
    worst = 0.0
    for tau in (0.0, 1e-3, 0.05, 1.0):
        t_d = t0.to(DEV)
        _check(L.sb200_soft_update_f32(_p(t_d), _p(s_d), n, tau, None, _st()), 'soft')
        torch.cuda.synchronize()
        keep = F32(1) - F32(tau)
        assert keep == F32(1.0 - tau)
        tn, sn = t0.numpy(), s.numpy()
        want = tn * keep + F32(tau) * sn
        got = t_d.cpu().numpy()
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), tau
        a64, b64 = tn.astype(np.float64) * (1 - tau), tau * sn.astype(np.float64)
        u = float((np.abs(got - (a64 + b64)) / _ulp(np.maximum(np.abs(a64), np.abs(b64)))).max())
        worst = max(worst, u)
        assert u <= SOFT_ULP_BAR, (tau, u)
    stop = torch.ones(1, dtype=torch.int32, device=DEV)
    t_d = t0.to(DEV)
    _check(L.sb200_soft_update_f32(_p(t_d), _p(s_d), n, 0.05, _p(stop), _st()), 'soft stop')
    torch.cuda.synchronize()
    assert torch.equal(t_d.cpu(), t0)
    print('measured soft', n, worst)


class PeriodicTracker:
    """The reference's session/tracker.py PeriodicTracker, restated: track_increment(incr) is True when the running
    value enters the next period."""

    def __init__(self, period, init_value=0, init_endpoint=0):
        self.period, self.value, self._endpoint = period, init_value, init_endpoint

    def track_increment(self, incr=1):
        self.value += incr
        if self.value >= self._endpoint + self.period:
            self._endpoint += (self.value - self._endpoint) // self.period * self.period
            return True
        return False


@pytest.mark.parametrize('period', [1, 3, 64, 150])
@pytest.mark.parametrize('incr', [1, 64])
def test_hard_update_follows_the_periodic_tracker(incr, period):
    """One sb200_hard_update_f32 per net per update, tick = 1 for the first net only, as the learners call it: the
    device counter equals PeriodicTracker.value after every update, each net is copied exactly on the updates where
    track_increment fires (the later nets on the same updates as the first), and an update with a raised stop flag
    neither ticks nor copies.  The run starts from 0 and again from a count left by an earlier run."""
    L = _lib_()
    sizes = [5, 1023, 264 * 1024 + 5]
    g = torch.Generator(device=DEV).manual_seed(incr * 1000 + period)
    steps = max(12, (5 * (2 * period + 7)) // (4 * incr) + 2)     # every fifth update is stopped
    for start in (0, 5 * incr):
        tr = PeriodicTracker(period, init_value=start, init_endpoint=start // period * period)
        counter = torch.tensor([start], dtype=torch.int64, device=DEV)
        tgt = [torch.randn(n, device=DEV, generator=g) for n in sizes]
        stop = torch.zeros(1, dtype=torch.int32, device=DEV)
        fired_any = 0
        for step in range(steps):
            src = [torch.randn(n, device=DEV, generator=g) for n in sizes]
            before = [t.clone() for t in tgt]
            stopped = step % 5 == 4
            stop.fill_(1 if stopped else 0)
            for i, (t, s) in enumerate(zip(tgt, src)):
                _check(L.sb200_hard_update_f32(_p(t), _p(s), t.numel(), _p(counter), period, incr, int(i == 0), _p(stop),
                                               _st()), 'hard')
            fire = False if stopped else tr.track_increment(incr)
            fired_any += fire
            assert int(counter.item()) == tr.value, (step, int(counter.item()), tr.value)
            for i, (t, s, b) in enumerate(zip(tgt, src, before)):
                assert torch.equal(t, s if fire else b), (start, step, i, fire)
        assert fired_any >= 2


# ------------------------------------------------------------------------------------------------------------------
# D. the weighted DDPG update against float64 autograd
W_GRAD_BAR, W_PRIO_BAR, W_STAT_BAR = 3e-5, 1.5e-5, 1e-7


@pytest.mark.parametrize('td3', [False, True])
def test_weighted_ddpg_learn_gradients(td3):
    """configs[2] (B 4096, D 64, A 8, actor 300-200, critic 400-300) and one weighted learn() (importance weights in
    [0.05, 1]): the pre-clip gradients of critic 1 (and critic 2 with TD3) against float64 autograd of
    mean(w (Q - y)^2) on the learner's own y, per tensor relative L2 / max error: measured worst 9.1e-6, bar
    W_GRAD_BAR = 3e-5.  The priorities |q1 - y| + eps come from critic 1 alone: error / max|q1| (the fp32 forward's
    error scale) measured worst 4.2e-6, bar W_PRIO_BAR = 1.5e-5.  td_error and avg_is_weight against float64,
    error / max(1, |v|): measured worst 2.8e-8, bar W_STAT_BAR = 1e-7."""
    from surreal_b200.learner import DDPGLearner
    D, A, B = 64, 8, 4096
    lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=(300, 200), critic_h=(400, 300), B=B, n_step=3, memory_size=8192,
                              start=B)
    lc.algo.network.use_double_critic = lc.algo.network.use_action_regularization = td3
    L = DDPGLearner(lc, ec, sc)
    gen = torch.Generator().manual_seed(21 + td3)
    al = _layers([D, 300, 200, A], gen)
    cls = [_layers([D, 400], gen) + _layers([400 + A, 300, 1], gen) for _ in range(2 if td3 else 1)]
    for m in (L.model, L.model_target):
        m.actor.load_layers(al)
        m.critic.load_layers(cls[0])
    if td3:
        for m in (L.model2, L.model_target2):
            m.critic.load_layers(cls[1])
    obs = torch.randn(B, D, generator=gen)
    act = torch.rand(B, A, generator=gen) * 2 - 1
    for _ in range(50):                                 # redraw rows with a float64 pre-activation within 2e-5 of 0
        bad = R.hidden_margin(obs, al) < 2e-5
        for cl in cls:
            bad |= R.hidden_margin(obs, cl, aux=act, aux_layer=1) < 2e-5
        if not bool(bad.any()):
            break
        obs[bad] = torch.randn(int(bad.sum()), D, generator=gen)
        act[bad] = torch.rand(int(bad.sum()), A, generator=gen) * 2 - 1
    assert not bool(bad.any())
    obs_next = torch.randn(B, D, generator=gen)
    rew, done = torch.randn(B, 1, generator=gen), (torch.rand(B, 1, generator=gen) < 0.05).float()
    w = torch.rand(B, generator=gen) * 0.95 + 0.05
    st = L.learn({'obs': obs.numpy(), 'obs_next': obs_next.numpy(), 'actions': act.numpy(), 'rewards': rew.numpy(),
                  'dones': done.numpy(), 'weights': w.numpy()})
    torch.cuda.synchronize()
    y = L._y.clone()
    rc = R.ddpg_critic(_dev(cls[0]), obs.to(DEV), act.to(DEV), y, weights=w)
    _check_grads(L.model.critic, L.critic_optim.grad, rc['grads'], 'weighted critic', bar=W_GRAD_BAR)
    if td3:
        rc2 = R.ddpg_critic(_dev(cls[1]), obs.to(DEV), act.to(DEV), y, weights=w)
        _check_grads(L.model2.critic, L.critic_optim2.grad, rc2['grads'], 'weighted critic 2', bar=W_GRAD_BAR)
    q1 = rc['q'].view(-1)
    d64 = q1 - R.f64(y).to(DEV)
    prio = L.td_priorities.double()
    e = (prio - (d64.abs() + L.priority_eps)).abs().max() / q1.abs().max()
    print('measured weighted prio', float(e))
    assert float(e) <= W_PRIO_BAR, float(e)
    for k, v in (('td_error', float(d64.abs().mean())), ('avg_is_weight', float(w.double().mean()))):
        err = abs(st[k] - v) / max(1.0, abs(v))
        print('measured weighted stat', k, err)
        assert err <= W_STAT_BAR, (k, st[k], v)


# ------------------------------------------------------------------------------------------------------------------
# E. a bad record first drawn in update k = 2 of K = 4
def _ddpg_state(L):
    ts = [L.model.actor.params, L.model.critic.params, L.model_target.actor.params, L.model_target.critic.params]
    opts = [L.actor_optim, L.critic_optim]
    if L.use_double_critic:
        ts += [L.model2.critic.params, L.model_target2.critic.params]
        opts.append(L.critic_optim2)
    for o in opts:
        ts += [o.exp_avg, o.exp_avg_sq, o.ws]
    return ts


def _dqn_state(L):
    ts = [n.params for n in L.model.nets() + L.model_target.nets()]
    for o in [L.optim_a] + ([L.optim_v] if L.dueling else []):
        ts += [o.exp_avg, o.exp_avg_sq, o.ws]
    return ts


def _tree(r):
    return [r.t_leaf, r.t_sum, r.t_min, r.ctrl, r.sampler]


def _clone(ts):
    return [t.clone() for t in ts]


def _load(ts, snap):
    for t, s in zip(ts, snap):
        t.copy_(s)


def _assert_same(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (what, i)


def _setup(algo, per):
    """-> (replay, learner A on graphs, twin learner B, state(learner), target counter attribute, batch size).  Both
    learners copy their targets every second update (DQN: every 2B samples), so update k = 2 would copy."""
    from surreal_b200.learner import DDPGLearner, DQNLearner
    learners = []
    if algo == 'ddpg':
        B = 16
        if per:
            r, _ = _per(600, D=9, A=3, B=B, sampler_seed=3, alpha=0.6, beta_anneal_iters=7)
            _fill_ring(r, 6)
            r.view.copy_(torch.tensor([590, 500, 600]))
        else:
            r, _ = _replay(600, D=9, A=3, B=B, sampler_seed=3)
            _set_view(r, 590, 500)
        for _ in range(2):
            lc, ec, sc = ddpg_configs(D=9, A=3, B=B, target={'type': 'hard', 'interval': 2})
            lc.algo.network.critic_regularization = 1e-3
            torch.manual_seed(11)
            learners.append(DDPGLearner(lc, ec, sc))
        state, attr = _ddpg_state, 'target_update_counter'
    else:
        B = 64
        lc, ec, sc = dqn_configs(B=B, period=2 * B, prioritized=per)
        r = _filled_replay(lc, ec, sc, per)
        for _ in range(2):
            torch.manual_seed(4)
            learners.append(DQNLearner(*dqn_configs(B=B, period=2 * B, prioritized=per)))
        state, attr = _dqn_state, 'target_update_samples'
    learners[0].use_cuda_graph = True
    return r, learners[0], learners[1], state, attr, B


def _hand_driven(r, LB, B, per, K):
    """K updates of LB, one learn() per batch, priorities written back by hand: -> the indices of each draw."""
    drawn = []
    for _ in range(K):
        b = r.sample_device(B, out=LB.replay_out_buffers())
        drawn.append(b['indices'].clone())
        LB.learn(b)
        if per:
            r.update_priorities(b['indices'], LB.td_priorities)
    torch.cuda.synchronize()
    return drawn


def _graph_vs_twin(r, LA, LB, state, attr, B, per, K):
    """One learn_from_replay(K) of LA against K hand-driven updates of LB from the same replay state."""
    snap = _clone(_tree(r)) if per else r.draw_counter
    sa = LA.learn_from_replay(r, updates=K)
    after = _clone(_tree(r)) if per else None
    if per:
        _load(_tree(r), snap)
    else:
        r.sampler[0] = snap
    _hand_driven(r, LB, B, per, K)
    if per:
        _assert_same(after, _tree(r), 'trees')
    _assert_same(state(LA), state(LB), 'learner')
    assert getattr(LA, attr) == getattr(LB, attr)
    return sa


@pytest.mark.parametrize('algo,per,bad', [('ddpg', False, 1.5), ('ddpg', False, NAN), ('ddpg', True, 1.5),
                                          ('ddpg', True, NAN), ('dqn', False, None), ('dqn', True, None)])
def test_bad_record_first_drawn_mid_call(algo, per, bad):
    """A bad record (a DDPG action component of 1.5 or NaN, a DQN action equal to n_actions) that is first drawn in
    update k = 2 of a K = 4 learn_from_replay call on a captured graph.  The rule: the call raises AssertionError;
    updates 1 .. k - 1 stand and update k and every later one of the call change nothing, so parameters, Adam moments
    and workspaces, targets, the target counter and the prioritized replay's trees equal a hand-driven twin after
    k - 1 updates, bit for bit; the replay's draw counters still advance by K (every sample launch drew).  Once the
    record is repaired, the next call continues exactly as the twin does from there."""
    K, k = 4, 2
    r, LA, LB, state, attr, B = _setup(algo, per)
    _graph_vs_twin(r, LA, LB, state, attr, B, per, K)     # a good call first: captures the graph, moves Adam
    snap_r = _clone(_tree(r)) if per else None
    c = r.draw_counter
    u = r.update_counter if per else None
    # the draws of updates 1 and 2: uniform from the sampler's restatement, prioritized from a hand-driven probe (that
    # path is bit-identical to the graph's) whose learner state is put back afterwards
    if per:
        snap_b, ctr_b = _clone(state(LB)), getattr(LB, attr)
        drawn = [d.cpu().numpy() for d in _hand_driven(r, LB, B, per, k)]
        _load(state(LB), snap_b)
        setattr(LB, attr, ctr_b)
        _load(_tree(r), snap_r)
    else:
        start, count, cap = r.view.tolist()
        drawn = [device_sample_indices(r.sampler_seed, c + j, start, count, cap, B) for j in range(k)]
    fresh = sorted(set(drawn[k - 1].tolist()) - set(np.concatenate(drawn[:k - 1]).tolist()))
    assert fresh, 'no record first drawn in update k'
    idx = fresh[0]
    col = 1 if algo == 'ddpg' else 0
    keep = float(r.r_act[idx, col])
    r.r_act[idx, col] = bad if algo == 'ddpg' else float(LA.n_actions)
    with pytest.raises(AssertionError):
        LA.learn_from_replay(r, updates=K)
    torch.cuda.synchronize()
    assert r.draw_counter == c + K
    if per:
        assert r.update_counter == u + K
    after_a = _clone(_tree(r)) if per else None
    # the twin: k - 1 updates from the same replay state
    if per:
        _load(_tree(r), snap_r)
    else:
        r.sampler[0] = c
    _hand_driven(r, LB, B, per, k - 1)
    _assert_same(state(LA), state(LB), 'learner after the failed call')
    assert getattr(LA, attr) == getattr(LB, attr)
    if per:
        _assert_same(after_a[:3], _tree(r)[:3], 'trees after the failed call')
        assert r.max_priority == float(after_a[3].view(torch.float32)[4])
        _load(_tree(r), after_a)                          # the replay as the failed call left it
    else:
        r.sampler[0] = c + K
    r.r_act[idx, col] = keep
    sa = _graph_vs_twin(r, LA, LB, state, attr, B, per, K)
    assert all(np.isfinite(v) for v in sa.values())

"""The batched n-step SSAR model (oracle.windowing.SsarBatch) against the reference's own wrapper: records and pending
float64 sums bit for bit on the multi-actor golden, the single-actor golden, and the single-actor model ssar_nstep.  The
GPU envelope test of the staging kernels takes this model as its oracle."""
from fractions import Fraction

import numpy as np
import pytest

from oracle.windowing import SsarBatch, ssar_nstep


def _bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


def _cases(golden):
    g = golden('window_ssar_multi')
    return g, g.js('cases')


def _drive(g, k, meta, capacity=None):
    """Run SsarBatch over case k; yields (t, model) after every step."""
    p = 'c%d/' % k
    N, T = meta['N'], meta['T']
    cap = capacity if capacity is not None else len(g[p + 'rec_rew']) + 7
    m = SsarBatch(N, meta['n_step'], meta['gamma'], cap)
    m.reset(list(g[p + 'obs0']))
    for t in range(T):
        m.step(list(g[p + 'action'][t]), list(g[p + 'obs_next'][t]), list(g[p + 'rew'][t]), list(g[p + 'done'][t]),
               obs_reset=list(g[p + 'obs_reset'][t]))
        yield t, m


def test_golden_covers_the_envelope(golden):
    g, cases = _cases(golden)
    assert sorted({c['n_step'] for c in cases}) == [1, 2, 3, 5]
    assert sorted({c['gamma'] for c in cases}) == [0.0, 0.37, 0.99, 1.0]
    for k, c in enumerate(cases):
        r = g['c%d/rew' % k]
        assert r.dtype == np.float64 and np.all(r.astype(np.float32).astype(np.float64) != r)   # not float32 values
        assert len(g['c%d/rec_rew' % k]) > 0


@pytest.mark.parametrize('k', range(16))
def test_batched_model_reproduces_the_reference_records_and_pending_sums(golden, k):
    g, cases = _cases(golden)
    meta = cases[k]
    p = 'c%d/' % k
    n = meta['n_step']
    for t, m in _drive(g, k, meta):
        for a in range(meta['N']):
            pend = m.pending(a)
            L = int(g[p + 'pend_len'][t, a])
            assert len(pend) == L, (t, a)
            assert [o for o, _, _ in pend] == list(g[p + 'pend_obs'][t, a, :L])
            assert [x for _, x, _ in pend] == list(g[p + 'pend_act'][t, a, :L])
            np.testing.assert_array_equal(_bits([s for _, _, s in pend]), g[p + 'pend_sum'][t, a, :L])
            assert L < n
    recs = m.ring.mem
    assert m.state() == (len(recs) % m.ring.memory_size, len(recs), m.ring.memory_size, len(recs))
    assert [r[0] for r in recs] == list(g[p + 'rec_obs'])
    assert [r[1] for r in recs] == list(g[p + 'rec_obs_next'])
    assert [r[2] for r in recs] == list(g[p + 'rec_act'])
    np.testing.assert_array_equal(_bits([r[3] for r in recs]), _bits(g[p + 'rec_rew']))
    assert [int(r[4]) for r in recs] == list(g[p + 'rec_done'])


def test_ring_overwrites_in_send_order(golden):
    """A ring smaller than the run: slot k % capacity holds the last record sent there; next_idx / size / total_in."""
    g, cases = _cases(golden)
    k = 10
    p = 'c%d/' % k
    total = len(g[p + 'rec_rew'])
    cap = 7
    for t, m in _drive(g, k, cases[k], capacity=cap):
        pass
    assert total > 2 * cap
    assert m.state() == (total % cap, cap, cap, total)
    for s in range(cap):
        last = max(j for j in range(total) if j % cap == s)
        assert m.ring.mem[s][0] == g[p + 'rec_obs'][last]
        assert _bits(m.ring.mem[s][3]) == _bits(g[p + 'rec_rew'][last])


def _fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def test_golden_tells_one_rounding_from_a_fused_multiply_add(golden):
    """Summing with one rounding (fma) instead of the reference's two gives different pending sums on this golden, so
    a kernel that contracts the accumulation cannot pass the tests built on it."""
    g, cases = _cases(golden)
    differ = 0
    for k, meta in enumerate(cases):
        p = 'c%d/' % k
        n, gamma = meta['n_step'], meta['gamma']
        fused = [[] for _ in range(meta['N'])]
        for t in range(meta['T']):
            for a in range(meta['N']):
                r = float(g[p + 'rew'][t, a])
                q = fused[a]
                for i in range(len(q)):
                    q[i] = _fma(pow(gamma, n - i - 1), r, q[i])
                q.append(r)
                if len(q) == n:
                    q.pop(0)
                if g[p + 'done'][t, a]:
                    q.clear()
                L = int(g[p + 'pend_len'][t, a])
                differ += int(np.sum(_bits(q) != g[p + 'pend_sum'][t, a, :L]))
    assert differ > 0


def test_single_actor_golden(golden):
    """The one-actor golden of make_golden.py (obs = step id, reward 0.25 g - 3) through the batched model."""
    for case in golden('window_ssar').js('cases'):
        n, gamma, ep_lens = case['n_step'], case['gamma'], case['ep_lens']
        m = SsarBatch(1, n, gamma, 1000)
        m.reset([0])
        g = 0
        for L in ep_lens:
            for t in range(L):
                m.step([float(g)], [g + 1], [0.25 * (g + 1) - 3.0], [t + 1 >= L])
                g += 1
        exp = case['records']
        assert [(r[0], r[1], r[2], r[4]) for r in m.ring.mem] == \
            [(e['obs'], e['obs_next'], e['action'], e['done']) for e in exp]
        assert [r[3] for r in m.ring.mem] == [e['reward'] for e in exp]


@pytest.mark.parametrize('n,gamma,ep_lens', [(1, 0.5, [3, 1, 2]), (3, 0.99, [7, 2, 5, 3]), (4, 0.37, [1, 9, 4, 6])])
def test_single_actor_agrees_with_ssar_nstep(n, gamma, ep_lens):
    rng = np.random.default_rng(n)
    rew = rng.standard_normal(sum(ep_lens) + 1) * 3.0
    m = SsarBatch(1, n, gamma, 1000)
    m.reset([0])
    g = 0
    for L in ep_lens:
        for t in range(L):
            m.step([g], [g + 1], [rew[g + 1]], [t + 1 >= L])
            g += 1
    exp = ssar_nstep(ep_lens, n, gamma, lambda i: float(rew[i]))
    assert [tuple(r) for r in m.ring.mem] == exp

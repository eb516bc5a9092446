"""Prioritized replay without a GPU: the float64 restatement in per_ref.py against the reference's own segment trees
(tests/golden/per_segment_tree.npz, made by tests/golden/make_golden_per.py), the view-restricted sampler, the
importance weights and beta schedule against the reference's formulas written literally, the ctypes binding of
sb200_per_tree, and the launcher flag.

Where the restatement departs from the reference's PrioritizedReplay (which cannot run as shipped), on purpose:
  * prioritized_replay.py:62-66 writes a new record's priority into the slot after it; here the record's own slot.
  * prioritized_replay.py:119 draws the mass from sum(0, len - 1), whose end is exclusive, so the newest record is never
    drawn; here the mass is the sum over the whole sampling view.
  * prioritized_replay.py:99-105 takes the minimum and N over the whole storage; here over the sampling view, the
    population the draw actually comes from (they coincide when the view is the whole ring)."""
import os

import numpy as np
import pytest

from per_ref import PerRef, TreeRef, beta_schedule, leaf_value, leaves_for, philox_u

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'per_segment_tree.npz')


@pytest.mark.parametrize('name', ['dyadic', 'random'])
def test_oracle_trees_match_the_reference_segment_trees(name):
    g = np.load(GOLDEN)
    leaf = g[name + '_leaf']
    t = TreeRef(50, leaf)
    assert t.P == 64
    assert np.array_equal(t.sum[1:], g[name + '_internal'][1:])          # pairwise parents: the same bits
    for (a, b), s, m in zip(g[name + '_ranges'], g[name + '_sums'], g[name + '_mins']):
        got = t.range_sum(int(a), int(b))
        if name == 'dyadic':
            assert got == s
        else:                                                             # another summation order: last bits only
            assert abs(got - s) <= 1e-14 * s
        assert float(t.range_min(int(a), int(b))) == m
    for x, want in zip(g[name + '_prefix'], g[name + '_found']):
        assert t.descend(float(x)) == want


def _random_tree(cap, seed):
    rng = np.random.RandomState(seed)
    leaf = np.zeros(leaves_for(cap), np.float32)
    leaf[:cap] = leaf_value(10.0 ** rng.uniform(-3, 1, size=cap), 0.6)
    return TreeRef(cap, leaf)


@pytest.mark.parametrize('cap,start,count', [(100, 0, 100), (100, 0, 37), (100, 20, 50), (100, 90, 60), (100, 99, 2),
                                             (1000, 700, 1000), (37, 36, 1), (2, 1, 2)])
def test_view_restricted_descent_stays_in_the_view(cap, start, count):
    t = _random_tree(cap, cap + start)
    us = np.concatenate([philox_u(5, 9, 4000), [0.0, 1.0 - 2.0 ** -53]])
    slots, _, S = t.sample(start, count, us)
    view = {(start + r) % cap for r in range(count)}
    assert set(slots.tolist()) <= view
    assert (t.leaf[slots] > 0).all()
    assert abs(S - sum(float(t.leaf[s]) for s in view)) <= 1e-12 * S
    likely = {s for s in view if float(t.leaf[s]) / S * len(us) > 20}
    assert likely <= set(slots.tolist())
    assert slots[-1] == (start + count - 1) % cap                         # the largest u lands on the newest record


def test_descent_is_proportional():
    from scipy.stats import chi2
    t = _random_tree(50, 3)
    us = philox_u(17, 0, 200000)
    slots, _, _ = t.sample(10, 45, us)
    view = [(10 + r) % 50 for r in range(45)]
    p = t.leaf[view].astype(np.float64)
    p /= p.sum()
    hist = np.array([(slots == s).sum() for s in view])
    stat = float(((hist - len(us) * p) ** 2 / (len(us) * p)).sum())
    assert stat < chi2.ppf(1 - 1e-4, len(view) - 1), stat


def test_weights_equal_the_reference_formula_written_literally():
    """prioritized_replay.py:98-105 over the view: p_min = min / sum, max_weight = (p_min * N)^-beta, and each weight
    (p_sample * N)^-beta / max_weight."""
    t = _random_tree(300, 8)
    start, count, beta = 250, 200, 0.55
    slots, _, _ = t.sample(start, count, philox_u(1, 2, 512))
    view = [(start + r) % 300 for r in range(count)]
    total = sum(float(t.leaf[s]) for s in view)
    p_min = min(float(t.leaf[s]) for s in view) / total
    max_weight = (p_min * count) ** (-beta)
    want = [((float(t.leaf[s]) / total) * count) ** (-beta) / max_weight for s in slots]
    got = t.weights(slots, start, count, beta)
    assert np.allclose(got, want, rtol=1e-12, atol=0)
    assert got.max() <= 1.0


def test_beta_schedule_matches_linear_schedule():
    """utils/schedule.py:96-99: LinearSchedule(schedule_timesteps, final_p=1.0, initial_p=beta0).value(t)."""
    def linear_schedule(t, schedule_timesteps, final_p, initial_p):
        fraction = min(float(t) / schedule_timesteps, 1.0)
        return initial_p + fraction * (final_p - initial_p)
    for t in (0, 1, 7, 99, 100, 101, 10 ** 6):
        assert beta_schedule(t, 0.4, 100) == linear_schedule(t, 100, 1.0, 0.4)
    assert beta_schedule(12345, 0.4, None) == 0.4


def test_admit_and_last_wins_update():
    r = PerRef(10, 0.6)
    r.admit(4)
    assert (r.tree.leaf[:4] == 1.0).all() and (r.tree.leaf[4:] == 0).all()
    r.update([2, 3, 2], [4.0, 0.5, 2.0])                                  # slot 2 ends with the last value
    assert r.tree.leaf[2] == leaf_value(2.0, 0.6) and r.tree.leaf[3] == leaf_value(0.5, 0.6)
    assert r.max_priority == 4.0
    r.admit(13)                                                           # 9 more inserts wrap the ring: slots 4..9, 0..2
    assert (r.tree.leaf[[4, 5, 6, 7, 8, 9, 0, 1, 2]] == leaf_value(4.0, 0.6)).all()
    assert r.tree.leaf[3] == leaf_value(0.5, 0.6)
    r.admit(40)                                                           # a gap of a whole ring or more: every slot
    assert (r.tree.leaf[:10] == leaf_value(4.0, 0.6)).all()
    assert r.tree.range_sum(0, 10) == r.tree.sum[1]


def test_tree_struct_binding_matches_the_header():
    """sb200_per_tree is declared with a tag: its fields against the ctypes binding, name by name."""
    import ctypes as C
    import re
    from surreal_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    txt = re.sub(r'/\*.*?\*/', '', open(os.path.join(root, 'include', 'surreal_b200.h')).read(), flags=re.S)
    body = re.search(r'typedef struct sb200_per_tree \{(.*?)\} sb200_per_tree;', txt, flags=re.S).group(1)
    fields = [re.match(r'\s*([\w ]+?)\s*(\**)\s*(\w+)\s*$', d).groups() for d in body.split(';') if d.strip()]
    assert [f[2] for f in fields] == [f[0] for f in _lib.PerTree._fields_]
    for (ctype, stars, _), (_, pytype) in zip(fields, _lib.PerTree._fields_):
        assert (pytype is C.c_void_p) == bool(stars)
        if not stars:
            assert ctype == 'int64_t' and pytype is C.c_int64


def test_launcher_flag_selects_prioritized_replay():
    from surreal_b200.main.ddpg_configs import ddpg_argparser
    base = ['--env', 'synthetic:12:4', '--num-agents', '4', '--experiment-folder', '/tmp/x']
    assert ddpg_argparser().parse_args(base + ['--prioritized-replay']).prioritized_replay
    assert not ddpg_argparser().parse_args(base).prioritized_replay

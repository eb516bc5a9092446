#!/usr/bin/env python
"""Generate the golden vectors of the prioritized replay's trees by running the REAL reference's segment trees
(surreal/replay/segment_tree.py, pure Python) on seeded priorities:

    python tests/golden/make_golden_per.py          # writes per_segment_tree.npz

  fixture                  reference code that produced it
  -----------------------  --------------------------------------------------------------------------------------------
  per_segment_tree.npz     SumSegmentTree / MinSegmentTree (segment_tree.py:6-138): __setitem__ of every leaf, then
                           sum(start, end), min(start, end) and find_prefixsum_idx(prefixsum)

Two leaf sets over a 64-leaf tree whose last 14 leaves are never set (a 50-slot ring): 'dyadic' holds multiples of 2^-8
(every sum is exact in any order, so range sums must match exactly), 'random' holds float32 p^0.6 of priorities spread
over four decades.  The leaves are set in a shuffled order, twice for some slots (the last value stays).  PrioritizedReplay
itself cannot run (it subclasses a Replay it never imports and reads an undefined _storage), so only its trees are pinned
here."""
import importlib.util
import os

import numpy as np

REF = '/root/reference/surreal/replay/segment_tree.py'
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'per_segment_tree.npz')
CAP, RING = 64, 50


def _segment_tree():
    spec = importlib.util.spec_from_file_location('segment_tree', REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    st = _segment_tree()
    rng = np.random.RandomState(2016)
    out = {}
    for name in ('dyadic', 'random'):
        if name == 'dyadic':
            leaf = rng.randint(1, 512, size=RING).astype(np.float32) / np.float32(256)
        else:
            p = 10.0 ** rng.uniform(-3, 1, size=RING)
            leaf = (p ** 0.6).astype(np.float32)
        ts, tm = st.SumSegmentTree(CAP), st.MinSegmentTree(CAP)
        order = rng.permutation(RING)
        again = rng.choice(RING, 10, replace=False)
        for i in again:                                          # set twice: the later value stays
            ts[int(i)] = 99.0
            tm[int(i)] = 99.0
        for i in order:
            ts[int(i)] = float(leaf[i])
            tm[int(i)] = float(leaf[i])
        ranges = [(0, RING), (0, 1), (5, 6), (3, 17), (16, 32), (7, 50), (31, 33), (49, 50), (0, 64), (20, 64)]
        sums = [ts.sum(a, b) for a, b in ranges]
        mins = [tm.min(a, b) for a, b in ranges]
        total = ts.sum()
        pref = np.concatenate([rng.uniform(0, total, size=200), [0.0, float(leaf[0]), float(leaf[0] + leaf[1])]])
        found = [ts.find_prefixsum_idx(float(x)) for x in pref]
        full = np.zeros(CAP, np.float32)
        full[:RING] = leaf
        out[name + '_leaf'] = full
        out[name + '_ranges'] = np.array(ranges, np.int64)
        out[name + '_sums'] = np.array(sums, np.float64)
        out[name + '_mins'] = np.array(mins, np.float64)
        out[name + '_prefix'] = pref.astype(np.float64)
        out[name + '_found'] = np.array(found, np.int64)
        out[name + '_internal'] = np.array(ts._value[:CAP], np.float64)
    np.savez(OUT, **out)
    print('wrote', OUT)


if __name__ == '__main__':
    main()

#!/usr/bin/env python
"""Bit-for-bit comparison of two `bench.py --dump-outputs DIR` directories: every .npy of the first must exist in the
second with the same shape, dtype and bytes (np.array_equal with NaN == NaN).  A change that must not alter numerics
(a schedule, an inlining, a work assignment) passes only if this does.

    python tools/compare_outputs.py DIR_A DIR_B        # exit status 0: identical; 1: a difference (listed)
"""
import glob
import os
import sys


def compare(dir_a, dir_b):
    import numpy as np
    names = sorted(os.path.basename(f) for f in glob.glob(os.path.join(dir_a, '*.npy')))
    if not names:
        print('no .npy files in %s' % dir_a)
        return False
    same = True
    for name in names:
        path_b = os.path.join(dir_b, name)
        if not os.path.exists(path_b):
            print('%-28s missing in %s' % (name, dir_b))
            same = False
            continue
        a, b = np.load(os.path.join(dir_a, name)), np.load(path_b)
        if a.shape != b.shape or a.dtype != b.dtype:
            print('%-28s shape / dtype %s %s vs %s %s' % (name, a.shape, a.dtype, b.shape, b.dtype))
            same = False
        elif not np.array_equal(a, b, equal_nan=True):
            n = int(np.sum(~((a == b) | (np.isnan(a) & np.isnan(b)))))
            print('%-28s %d of %d elements differ, max |a - b| %.3g' % (name, n, a.size, float(np.nanmax(np.abs(a - b)))))
            same = False
    extra = sorted(set(os.path.basename(f) for f in glob.glob(os.path.join(dir_b, '*.npy'))) - set(names))
    for name in extra:
        print('%-28s only in %s' % (name, dir_b))
        same = False
    print('%d arrays: %s' % (len(names), 'bit-identical' if same else 'DIFFERENT'))
    return same


if __name__ == '__main__':
    if len(sys.argv) != 3:
        raise SystemExit(__doc__)
    sys.exit(0 if compare(sys.argv[1], sys.argv[2]) else 1)

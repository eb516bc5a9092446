"""The one-launch learner kernel's plan does not depend on its grid: the weight-gradient row split (s, rows per split) and
the squared-norm chunking are sized for one CTA per SM, so a learner whose grid is capped to the SMs the actors leave free
computes the same sums in the same order.  Host code behind the C-ABI; no GPU needed."""
from surreal_b200 import ops

from test_epoch_plan import _block


def _plan(shapes, grid):
    (pd, pmode, M), (vd, vmode, _) = shapes
    p, v = _block(pd, pmode, M=M), _block(vd, vmode, M=M)
    p.args.grid = grid
    return ops.EpochPair.plan(p, v)


def test_plan_is_the_same_at_any_grid():
    cases = [
        (([64, 256, 256, 8], 0, 1024), ([64, 256, 256, 1], 2, 1024)),     # the bench shape
        (([64, 256, 256, 8], 1, 4096), ([64, 256, 256, 1], 2, 4096)),
        (([17, 300, 200, 6], 0, 200), ([17, 100, 68, 1], 2, 200)),         # ragged
    ]
    for shapes in cases:
        full = _plan(shapes, 0)
        assert full['grid'] >= 37 and full['norm_chunks'] == full['grid']
        for grid in (full['grid'], 68, 37, 1):
            pl = _plan(shapes, grid)
            assert pl['grid'] == grid
            assert {k: v for k, v in pl.items() if k != 'grid'} == {k: v for k, v in full.items() if k != 'grid'}, (shapes, grid)

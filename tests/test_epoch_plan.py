"""Host side of the one-launch learner kernel (csrc/epoch2.cu): the shared-memory / work plan that decides whether a pair of
networks is taken by the kernel or falls back to the launch chain, and the workspace it asks for.  No GPU needed: planning is
host code behind the C-ABI (`sb200_ppo_epochs2_supported`, `sb200_ppo_epochs2_workspace_bytes`)."""
import ctypes as C

import torch

from surreal_b200 import _lib, ops


def _block(dims, mode, M=1024):
    acts = [ops.ACT_RELU] * (len(dims) - 2) + [ops.ACT_TANH if mode != 2 else ops.ACT_NONE]
    net = ops.FlatNet(dims, acts, 'cpu', extra=(dims[-1] if mode != 2 else 0))
    tr = ops.MlpTrainer(net, M, 1e-4)
    x, stats = torch.zeros(M, dims[0]), torch.zeros(32)
    if mode != 2:
        A = dims[-1]
        return ops.EpochKernel(tr, mode, x, dims[0], M, None, 1e-2, stats, 10, actions=torch.zeros(M, A), lda=A,
                               adv=torch.zeros(M), behave_pd=torch.zeros(M, 2 * A), ldb=2 * A, ref_pd=torch.zeros(M, 2 * A),
                               ldr=2 * A, hyper=torch.zeros(2, dtype=torch.float64), grid=148)
    return ops.EpochKernel(tr, 2, x, dims[0], M, None, 1e-2, stats, 10, returns=torch.zeros(M), grid=148)


def _ws(p, v):
    return int(_lib.lib().sb200_ppo_epochs2_workspace_bytes(C.byref(p.args), C.byref(v.args) if v is not None else None))


def test_bench_shape_is_taken_and_workspace_scales_with_the_batch():
    p, v = _block([64, 256, 256, 8], 0), _block([64, 256, 256, 1], 2)
    assert ops.EpochPair.supported(p, v)
    assert ops.EpochPair.supported(p, None)                      # a single optimiser is a valid launch too
    small = _ws(p, v)
    p4, v4 = _block([64, 256, 256, 8], 1, M=4096), _block([64, 256, 256, 1], 2, M=4096)
    assert ops.EpochPair.supported(p4, v4)
    big = _ws(p4, v4)
    # per row block (16 rows) and network: KL partial + loss partials + the dW3 partial ((H2 + 1) * ru4(out) floats)
    assert big > small > 2 * 256 * 256 * 4                       # at least the two transposed W2 copies
    assert big - small >= (4096 - 1024) // 16 * ((256 + 1) * 8 * 4)


def test_ragged_shapes_are_taken():
    assert ops.EpochPair.supported(_block([17, 300, 200, 6], 0, M=200), _block([17, 100, 68, 1], 2, M=200))
    assert ops.EpochPair.supported(_block([20, 64, 64, 1], 1, M=77), _block([20, 64, 64, 1], 2, M=77))


def test_shapes_the_kernel_rejects_fall_back():
    v = _block([64, 256, 256, 1], 2)
    assert not ops.EpochPair.supported(_block([64, 600, 256, 8], 0), v)          # wider than the shared-memory plan allows
    assert not ops.EpochPair.supported(_block([64, 256, 256, 40], 0), v)         # head wider than 32
    four = ops.FlatNet([64, 128, 128, 128, 8], [ops.ACT_RELU] * 3 + [ops.ACT_TANH], 'cpu', extra=8)
    assert four.n_layers == 4                                                    # PPOLearner._epoch_kernels screens these out


# ---- the plan's edges, against a restatement of e2_plan -------------------------------------------------------------
RB, MAX_OUT, MAX_WIDTH = 16, 32, 512
SMEM_FLOATS = 220 * 1024 // 4


def _ru4(v):
    return (v + 3) & ~3


def _mirror(jobs, G, max_width=MAX_WIDTH):
    """e2_plan restated: ``jobs`` = [(dims, M, splits)] -> [(s, rps)] per job, or None when the pair is rejected.  The
    activation region (16 rows of x, h1, h2, d2, head, dpre) doubles as the A operand of the weight-gradient items
    (16 x (rps + 4)); then the GEMM partials (4 x 17 rows of the widest layer), W3 and the per-row loss operands."""
    for dims, _, _ in jobs:
        if len(dims) != 4 or min(dims) < 1 or dims[3] > MAX_OUT or max(dims[:3]) > max_width:
            return None
    ld_xs = max([4] + [_ru4(d[0]) for d, _, _ in jobs])
    ld_h1 = max([4] + [_ru4(d[1]) for d, _, _ in jobs])
    ld_h2 = max([4] + [_ru4(d[2]) for d, _, _ in jobs])
    max_w3 = max([4] + [d[2] * _ru4(d[3]) for d, _, _ in jobs])
    blocks = sum(-(-d[1] // RB) + -(-d[0] // RB) + 1 for d, _, _ in jobs)
    out, max_as = [], 0
    for _, M, splits in jobs:
        s = min(max(1, G // blocks), splits, max(1, M // 64))
        rps = _ru4(-(-M // s))
        out.append((s, rps))
        max_as = max(max_as, RB * (_ru4(rps) + 4))
    act = RB * (ld_xs + ld_h1 + 2 * ld_h2 + 2 * MAX_OUT)
    off = max(act, _ru4(max_as)) + 4 * (RB + 1) * max(ld_h1, ld_h2) + _ru4(max_w3) + RB * (5 * MAX_OUT + 1)
    return out if off <= SMEM_FLOATS else None


def _plan_sms():
    """SMs the plan is sized for (the device's, or 132 without one)."""
    p, v = _block([64, 256, 256, 8], 0), _block([64, 256, 256, 1], 2)
    return ops.EpochPair.plan(p, v)['norm_chunks']


def _at_rows(blocks, M):
    """Re-point the plan inputs of EpochKernel blocks at M rows with MlpTrainer's default row splits (planning only: the
    buffers behind them are not touched)."""
    for b in blocks:
        b.args.M, b.args.splits = M, max(1, min(16, M // 128))
    return blocks


def _jobs(blocks):
    return [(list(C.cast(b.args.net, C.POINTER(_lib.Mlp)).contents.dims)[:4], b.args.M, b.args.splits) for b in blocks]


def _accepts(blocks):
    return ops.EpochPair.supported(*blocks)


def _last_true(ok, lo, hi):
    """Largest v in [lo, hi) with ok(v), given ok(lo) and not ok(hi)."""
    assert ok(lo) and not ok(hi), (lo, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if ok(mid) else (lo, mid)
    return lo


def _pair_blocks(H1, H2, D=64, A=8, M=1024, mode=0):
    return [_block([D, H1, H2, A], mode, M=M), _block([D, H1, H2, 1], 2, M=M)]


def largest_rows(H1=256, H2=256, D=64, A=8):
    """Largest batch the kernel takes for this pair of networks (MlpTrainer's default splits), by bisection."""
    blocks = _pair_blocks(H1, H2, D, A)
    return _last_true(lambda M: _accepts(_at_rows(blocks, M)), 2, 1 << 20)


def widest_square(M=1024, D=64, A=8):
    """Widest H the kernel takes for D-H-H-A / D-H-H-1 at M rows, by bisection."""
    return _last_true(lambda H: _accepts(_at_rows(_pair_blocks(H, H, D, A), M)), 4, MAX_WIDTH + 1)


def test_plan_matches_its_restatement():
    """Acceptance, row splits and rows per split of the library's plan equal _mirror's at shapes on both sides of every
    width, head and row edge: a change to the plan has to change the restatement with it."""
    G = _plan_sms()
    nets = [([17, 15, 17, 5], [17, 16, 15, 1]), ([3, 257, 260, 9], [3, 256, 257, 1]), ([16, 416, 416, 8], [16, 416, 416, 1]),
            ([64, 420, 416, 8], [64, 416, 416, 1]), ([64, 256, 256, 32], [64, 256, 256, 1]),
            ([64, 256, 256, 33], [64, 256, 256, 1]), ([512, 16, 16, 4], [512, 16, 16, 1]),
            ([513, 16, 16, 4], [513, 16, 16, 1]), ([8, 513, 8, 4], [8, 8, 8, 1]), ([8, 8, 512, 1], [8, 8, 8, 1])]
    seen = [0, 0]
    for pd, vd in nets:
        blocks = [_block(pd, 0, M=256), _block(vd, 2, M=256)]
        for M in (2, 3, 16, 63, 64, 127, 128, 129, 255, 256, 577, 1000, 1024, 4096, 6408, 6409, 9000):
            _at_rows(blocks, M)
            exp = _mirror(_jobs(blocks), G)
            assert _accepts(blocks) == (exp is not None), (pd, vd, M, exp)
            seen[exp is not None] += 1
            if exp is not None:
                pl = ops.EpochPair.plan(*blocks)
                assert [(pl['s'][j], pl['rps'][j]) for j in range(2)] == exp, (pd, vd, M, pl, exp)
    assert min(seen) >= 20, seen


def test_plan_limits():
    """The edges the GPU envelope test runs at, found by bisection and pinned to the restatement: the bench shape's
    largest batch, the widest square hidden layers at 1024 rows and those networks' largest batch.  Widths past 512 and
    heads past 32 are rejected by the width rule, not only by the shared-memory budget."""
    G = _plan_sms()
    m_bench = largest_rows()
    assert _mirror([([64, 256, 256, 8], m_bench, max(1, min(16, m_bench // 128))),
                    ([64, 256, 256, 1], m_bench, max(1, min(16, m_bench // 128)))], G) is not None
    m1 = m_bench + 1
    assert _mirror([([64, 256, 256, 8], m1, max(1, min(16, m1 // 128))), ([64, 256, 256, 1], m1, max(1, min(16, m1 // 128)))], G) is None
    assert m_bench >= 4096, m_bench                              # every bench batch size (1024 and 4096) is taken
    h = widest_square()
    assert 256 <= h < MAX_WIDTH, h                               # the shared-memory budget binds before the width rule
    assert _accepts(_pair_blocks(h, h)) and not _accepts(_pair_blocks(h + 1, h + 1))
    m_wide = largest_rows(h, h)
    assert 1024 <= m_wide < m_bench, (m_wide, m_bench)
    # the width rule: 512 wide inputs are taken, 513 are not, although the budget would have room for them
    wide_in = [([513, 16, 16, 4], 256, 2), ([513, 16, 16, 1], 256, 2)]
    assert _accepts(_at_rows([_block([512, 16, 16, 4], 0, M=256), _block([512, 16, 16, 1], 2, M=256)], 256))
    assert not _accepts(_at_rows([_block([513, 16, 16, 4], 0, M=256), _block([513, 16, 16, 1], 2, M=256)], 256))
    assert _mirror(wide_in, G) is None and _mirror(wide_in, G, max_width=1024) is not None
    assert _accepts([_block([64, 256, 256, 32], 0), _block([64, 256, 256, 1], 2)])
    print('plan limits at %d SMs: bench shape M <= %d, square H <= %d at 1024 rows, M <= %d at H = %d' % (G, m_bench, h, m_wide, h))

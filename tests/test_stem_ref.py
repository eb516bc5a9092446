"""The float64 stem reference of tests/stem_ref.py on the CPU: it agrees with torch's own float32 convolutions, its
envelope mirror reproduces the shared-memory limits of csrc/stem.cu, and the exact-operand builders' preconditions hold
at every shape tests/test_stem_envelope_gpu.py runs."""
import pytest
import torch
import torch.nn.functional as F

import stem_ref as R
from surreal_b200.main.ppo_configs import PPO_DEFAULT_LEARNER_CONFIG as LC

ROWS = dict(zip(('M', 'ALL'), R.learner_rows(LC.replay.batch_size, LC.algo.n_step, LC.algo.rnn.horizon)))


@pytest.mark.parametrize('layer,C,H,W', [(1, 3, 20, 27), (1, 1, 8, 8), (2, 16, 9, 12), (2, 5, 4, 7)])
def test_reference_matches_float32_torch(layer, C, H, W):
    """Forward, dW / db and dX against float32 F.conv2d + autograd in torch's weight layout; every result within
    the a-priori bound of its own chain, and |reference| <= sum |terms|."""
    KS, ST, CO = R.LAYERS[layer]
    g = torch.Generator().manual_seed(layer * 1000 + C * 100 + H + W)
    n, scale = 3, 1.0 / 255.0 if layer == 1 else 1.0
    x = torch.randint(0, 256, (n, C, H, W), generator=g).float() if layer == 1 else torch.relu(torch.randn(n, C, H, W, generator=g))
    w = torch.randn(CO, C, KS, KS, generator=g) * 0.1
    b = torch.randn(CO, generator=g) * 0.1
    Wk = R.to_kernel(w)
    assert torch.equal(R.to_torch(Wk, C, layer), w)
    xin = (x * scale).requires_grad_(True)
    wt, bt = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    pre = F.conv2d(xin, wt, bt, stride=ST)
    dy = torch.randn(pre.shape, generator=g) * (pre > 0)
    pre.backward(dy)
    act = torch.relu(torch.randn(n, C, H, W, generator=g))

    def within(got32, ref64, S, K):
        assert ref64.dtype == torch.float64 and bool((ref64.abs() <= S * (1 + 1e-12)).all())
        # float32 torch sums the same terms in its own order, a summation tree at most K + 1 deep
        assert bool(((got32.double() - ref64).abs() <= R.bound(S, K + 1)).all())

    within(torch.relu(pre.detach()), R.forward(x, Wk, b, scale, layer), R.abs_forward(x, Wk, b, scale, layer),
           R.chain_fwd(layer, C))
    gw, gb = R.weight_grad(x, dy, scale, layer)
    sw, sb = R.abs_weight_grad(x, dy, scale, layer)
    K = R.chain_dw(layer, n, 1, H, W)
    within(R.to_kernel(wt.grad), gw, sw, K)
    within(bt.grad, gb, sb, K)
    if layer == 2:
        within(xin.grad * (act > 0), R.input_grad(dy, Wk, act, C, H, W), R.abs_input_grad(dy, Wk, C, H, W), R.chain_dx())
        assert torch.equal(R.input_grad(dy, Wk, None, C, H, W) * (act > 0), R.input_grad(dy, Wk, act, C, H, W))


def test_exact_operands_give_exact_reference():
    """On builder operands the float64 results are integer multiples of their unit q below 2^24 q."""
    g = torch.Generator().manual_seed(3)
    x, Wk, b, s = R.fwd_operands(g, 1, 2, 4, 20, 24, 'cpu')
    y = R.forward(x, Wk, b, s, 1)
    assert torch.equal(y, torch.round(y * 64) / 64) and float(y.abs().max()) * 64 < R.EXACT_LIMIT
    x, dy, s = R.dw_operands(g, 2, 5, 16, 9, 11, 'cpu')
    gw, gb = R.weight_grad(x, dy, s, 2)
    assert torch.equal(gw, torch.round(gw * 16) / 16) and torch.equal(gb, torch.round(gb))
    assert bool((dy != 0).sum((2, 3)).eq(R.dw_nz(2, 5, 9, 11, 255)).all())


def test_envelope_mirror_limits():
    """launch_fwd / launch_dw / sb200_conv_backward_dx_f32 refuse more than 200 KB of dynamic shared memory.  At 84x84
    the forward takes C <= 5 and dW C <= 6, so a C = 6 frame stack is refused by the forward alone; one-channel square
    frames reach 212 px in the forward but 163 px in dW; four channels 98 and 102 px."""
    for layer, kind, C, H, W, axis, top in R.ENVELOPE_CASES:
        assert R.largest(layer, kind, C, H, W, axis) == top, (layer, kind, axis)
    assert R.accepts(1, 'dw', 6, 84, 84) and not R.accepts(1, 'fwd', 6, 84, 84)
    assert R.envelope(2, 'fwd', 16, 84, 20) == R.SMEM_MAX               # exactly at the limit is accepted
    # the default stem: 84x84x4 frames, conv2 on conv1's 16 x 20 x 20 output
    assert R.envelope(1, 'fwd', 4, 84, 84) == 4 * (4 * 64 * 16 + 4 * 84 * 104)
    assert R.envelope(1, 'dw', 4, 84, 84) == 4 * (4 * 84 * 84 + 400 * 16)
    assert R.envelope(2, 'dx', 16, 20, 20) == 4 * (16 * 16 * 32 + 81 * 32)


def test_builder_preconditions_at_gpu_shapes():
    """Every exact case of the GPU test builds (the builders assert the 2^24 condition), the learner's frame counts
    included; the dW cases at those counts get a dy dense enough to reach every weight."""
    g = torch.Generator().manual_seed(0)
    assert ROWS == {'M': 1344, 'ALL': 1664}
    for _, layer, frames, C, H, W, opts in R.FWD_CASES:
        n, _ = R.resolve(frames, 1, ROWS)
        R.fwd_operands(g, layer, min(n, 2), C, H, W, 'cpu', **opts)        # the condition does not depend on frames
    for _, layer, frames, C, H, W, splits, opts in R.DW_CASES:
        n, _ = R.resolve(frames, splits, ROWS)
        R.dw_operands(g, layer, n, C, H, W, 'cpu', **opts)
        HO, WO = R.out_hw(layer, H, W)
        assert n * R.dw_nz(layer, n, H, W, opts.get('fill', 255)) >= HO * WO, 'dy too sparse to reach every position'
    for _, frames, C, H, W in R.DX_CASES:
        R.dx_operands(g, 2, C, H, W, 'cpu')
    for layer, kind, C, H, W, axis, top in R.ENVELOPE_CASES:
        shape = dict(C=(top, H, W), H=(C, top, W), W=(C, H, top), HW=(C, top, top))[axis]
        if kind == 'fwd':
            R.fwd_operands(g, layer, 1, *shape, 'cpu')
        elif kind == 'dw':
            R.dw_operands(g, layer, 2, *shape, 'cpu')

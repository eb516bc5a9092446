"""The CNN stem convolutions (csrc/stem.cu) against float64 (tests/stem_ref.py) at the pixel learner's frame counts,
around the forward / dX grid cap, at every masked or partial path, and at the edges of their shared-memory envelope.

a. Exact: integer-valued operands make every fp32 product and partial sum exact, so y == y64 bit for bit (-0 == 0); a
   wrong tap, frame, channel, slab or mask is a mismatch.  dW is checked slab by slab (slab z = frames z, z + splits, ...)
   and summed.  Case ids name the path: grid_stride (frames past 528 CTAs), masked_col_group (WO % 4), tap_batch2
   (C * KS^2 > 256 taps), idle_slabs (splits > frames), ho1 / wo1, learner_* (the default pixel learner's rows).
b. Bounded: learner-like values (x / 255, torch's default Conv2d initialisation, Gaussian dy masked by relu'),
   |y - y64| <= bound(sum |terms|, K) for each kernel's longest fp32 chain K (stem_ref.bound).
c. Envelope: at the largest accepted size along C, H and W each launch returns SB200_OK and is exact; one step past it
   returns SB200_ERR_UNSUPPORTED and leaves its NaN-filled outputs untouched.
d. One StemTrainer backward at the default pixel shapes, each stage against float64 on the stage's own fp32 inputs."""
import ctypes
import zlib

import pytest
import torch

import stem_ref as R
from surreal_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NAN = float('nan')
OK, ERR_ARG, ERR_UNSUPPORTED = 0, -1, -3


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _lib_():
    ops._stream()                     # sb200_init once
    return _lib.lib()


def _gen(tag):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(tag).encode()))


@pytest.fixture(scope='module')
def rows(tmp_path_factory):
    """update rows M = B * eff_len and critic rows B * (n + 1) of a default-config PPOLearner on [4, 84, 84] frames"""
    import copy
    from surreal_b200.session import Config
    from surreal_b200.main.ppo_configs import (PPO_DEFAULT_LEARNER_CONFIG, PPO_DEFAULT_ENV_CONFIG, PPO_DEFAULT_SESSION_CONFIG,
                                               make_synthetic_pixel_env_config)
    from surreal_b200.learner import PPOLearner
    lc, ec, sc = (Config(copy.deepcopy(c.to_dict())) for c in (PPO_DEFAULT_LEARNER_CONFIG, PPO_DEFAULT_ENV_CONFIG,
                                                                 PPO_DEFAULT_SESSION_CONFIG))
    sc.folder = str(tmp_path_factory.mktemp('pixel_learner'))
    lc.algo.use_z_filter = False                        # frames alone: nothing to filter
    make_synthetic_pixel_env_config(ec, 64, frame_shape=(4, 84, 84), action_dim=6)
    ch = PPOLearner(lc, ec, sc).chain
    out = {'M': ch.M, 'ALL': ch.B * ch.n1}
    del ch
    torch.cuda.empty_cache()
    return out


# ---- launches ------------------------------------------------------------------------------------------------------
def _fwd(layer, x, Wk, b, s, frames=None):
    n, C, H, W = x.shape
    n = n if frames is None else frames
    HO, WO = R.out_hw(layer, H, W)
    y = torch.full((max(n, 1), R.LAYERS[layer][2], HO, WO), NAN, device=DEV)
    rc = _lib_().sb200_conv_forward_f32(layer, _p(x), int(x.dtype == torch.uint8), n, C, H, W, _p(Wk), _p(b), s, _p(y),
                                        ops._stream())
    torch.cuda.synchronize()
    return rc, y


def _dw(layer, x, dy, s, splits):
    """-> rc, slabs_w [splits, taps, COUT], slabs_b [splits, COUT], guard [splits, 4] (NaN-filled beforehand)"""
    n, C, H, W = x.shape
    KS, _, CO = R.LAYERS[layer]
    nw = C * KS * KS * CO
    stride = nw + CO + 4
    slabs = torch.full((splits, stride), NAN, device=DEV)
    rc = _lib_().sb200_conv_backward_dw_f32(layer, _p(x), int(x.dtype == torch.uint8), _p(dy), n, C, H, W, s, _p(slabs),
                                            ctypes.c_void_p(slabs.data_ptr() + 4 * nw), stride, splits, ops._stream())
    torch.cuda.synchronize()
    return rc, slabs[:, :nw].view(splits, -1, CO), slabs[:, nw:nw + CO], slabs[:, nw + CO:]


def _dx(dy, Wk, act, C, H, W):
    n = dy.shape[0]
    dx = torch.full((n, C, H, W), NAN, device=DEV)
    rc = _lib_().sb200_conv_backward_dx_f32(2, _p(dy), _p(Wk), _p(act), n, C, H, W, _p(dx), ops._stream())
    torch.cuda.synchronize()
    return rc, dx


def _exact(got, ref, what):
    bad = int((got.double() != ref).sum())          # NaN (unwritten) counts; -0.0 == 0.0
    print('measured mismatches', what, bad, 'of', ref.numel())
    assert bad == 0, (what, bad)


def _slab_refs(layer, x, dy, s, splits):
    """float64 partial (dWk, db) of each slab: frames z, z + splits, ... (zeros for a CTA that gets no frame)"""
    KS, _, CO = R.LAYERS[layer]
    out = []
    for z in range(splits):
        if z < x.shape[0]:
            out.append(R.weight_grad(x[z::splits], dy[z::splits], s, layer))
        else:
            out.append((torch.zeros(x.shape[1] * KS * KS, CO, dtype=torch.float64, device=DEV),
                        torch.zeros(CO, dtype=torch.float64, device=DEV)))
    return out


def _frames(frames, request):
    return request.getfixturevalue('rows')[frames] if isinstance(frames, str) else frames


# ---- a. exact ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', R.FWD_CASES, ids=[c[0] for c in R.FWD_CASES])
def test_forward_exact(case, request):
    tag, layer, frames, C, H, W, opts = case
    n = _frames(frames, request)
    x, Wk, b, s = R.fwd_operands(_gen(('fwd', tag)), layer, n, C, H, W, DEV, **opts)
    rc, y = _fwd(layer, x, Wk, b, s)
    assert rc == OK
    _exact(y, R.forward(x, Wk, b, s, layer), ('fwd', tag, n))


@pytest.mark.parametrize('case', R.DW_CASES, ids=[c[0] for c in R.DW_CASES])
def test_weight_grad_exact_per_slab(case, request):
    tag, layer, frames, C, H, W, splits, opts = case
    n, splits = R.resolve(_frames(frames, request), splits, {})
    x, dy, s = R.dw_operands(_gen(('dw', tag)), layer, n, C, H, W, DEV, **opts)
    rc, sw, sb, guard = _dw(layer, x, dy, s, splits)
    assert rc == OK
    assert bool(torch.isnan(guard).all()), 'written past the bias slab'
    for z, (gw, gb) in enumerate(_slab_refs(layer, x, dy, s, splits)):
        _exact(sw[z], gw, ('dw slab', tag, z))
        _exact(sb[z], gb, ('db slab', tag, z))
    gw, gb = R.weight_grad(x, dy, s, layer)
    _exact(sw.double().sum(0), gw, ('dw', tag, n, splits))
    _exact(sb.double().sum(0), gb, ('db', tag, n, splits))


@pytest.mark.parametrize('case', R.DX_CASES, ids=[c[0] for c in R.DX_CASES])
def test_input_grad_exact(case, request):
    """with act (the relu' mask drops exact zeros) and with act = NULL (no mask)"""
    tag, frames, C, H, W = case
    n = _frames(frames, request)
    dy, Wk, act = R.dx_operands(_gen(('dx', tag)), n, C, H, W, DEV)
    assert bool((act == 0).any())
    for a in (act, None):
        rc, dx = _dx(dy, Wk, a, C, H, W)
        assert rc == OK
        _exact(dx, R.input_grad(dy, Wk, a, C, H, W), ('dx', tag, n, 'act' if a is not None else 'no act'))


# ---- b. bounded, learner-like values -------------------------------------------------------------------------------
def _ratio(got, ref, S, K):
    """max |got - ref| / bound over all outputs (an output with S = 0 must be exact)"""
    err = (got.double() - ref).abs()
    return float((err / R.bound(S, K).clamp_min(1e-300)).max())


@pytest.mark.parametrize('which', ['M', 'ALL'])
def test_learner_values_within_bound(which, rows):
    """Both convolutions, dW slab by slab and summed, and dX at the learner's rows with real values: frames / 255
    (1/255 rounded to fp32, then the product rounded), torch's default Conv2d initialisation, N(0, 1) dy masked by
    relu' of the kernel's own forward."""
    n = rows[which]
    splits = max(1, min(16, n // 16))
    g = _gen(('bounded', n))
    torch.manual_seed(n)
    c1, c2 = torch.nn.Conv2d(4, 16, 8, 4), torch.nn.Conv2d(16, 32, 4, 2)
    Wk1, b1 = R.to_kernel(c1.weight.detach()).to(DEV), c1.bias.detach().to(DEV)
    Wk2, b2 = R.to_kernel(c2.weight.detach()).to(DEV), c2.bias.detach().to(DEV)
    x = torch.randint(0, 256, (n, 4, 84, 84), generator=g, device=DEV, dtype=torch.uint8)
    s = 1.0 / 255.0
    ratios = {}
    rc, a1 = _fwd(1, x, Wk1, b1, s)
    assert rc == OK
    ratios['fwd1'] = _ratio(a1, R.forward(x, Wk1, b1, s, 1), R.abs_forward(x, Wk1, b1, s, 1), R.chain_fwd(1, 4))
    rc, a2 = _fwd(2, a1, Wk2, b2, 1.0)
    assert rc == OK
    ratios['fwd2'] = _ratio(a2, R.forward(a1, Wk2, b2, 1.0, 2), R.abs_forward(a1, Wk2, b2, 1.0, 2), R.chain_fwd(2, 16))
    for layer, xin, y, sc, H in ((1, x, a1, s, 84), (2, a1, a2, 1.0, 20)):
        dy = torch.randn(y.shape, generator=g, device=DEV) * (y > 0)
        rc, sw, sb, _ = _dw(layer, xin, dy, sc, splits)
        assert rc == OK
        for z, (gw, gb) in enumerate(_slab_refs(layer, xin, dy, sc, splits)):
            aw, ab = R.abs_weight_grad(xin[z::splits], dy[z::splits], sc, layer)
            K = R.chain_dw(layer, len(range(z, n, splits)), 1, H, H)
            ratios['dw%d_slab' % layer] = max(ratios.get('dw%d_slab' % layer, 0.0), _ratio(sw[z], gw, aw, K),
                                             _ratio(sb[z], gb, ab, K))
        gw, gb = R.weight_grad(xin, dy, sc, layer)
        aw, ab = R.abs_weight_grad(xin, dy, sc, layer)
        K = R.chain_dw(layer, n, splits, H, H)
        ratios['dw%d_sum' % layer] = max(_ratio(sw.double().sum(0), gw, aw, K), _ratio(sb.double().sum(0), gb, ab, K))
        if layer == 2:
            rc, dx = _dx(dy, Wk2, a1, 16, 20, 20)
            assert rc == OK
            ratios['dx'] = _ratio(dx, R.input_grad(dy, Wk2, a1, 16, 20, 20), R.abs_input_grad(dy, Wk2, 16, 20, 20),
                                  R.chain_dx())
    print('measured bound ratio', which, n, ratios)
    assert all(r <= 1.0 for r in ratios.values()), ratios


# ---- c. envelope ---------------------------------------------------------------------------------------------------
def _run(layer, kind, C, H, W, tag):
    """one exact call of `kind` at [2, C, H, W] -> (rc, outputs, references)"""
    g = _gen((kind, tag))
    if kind == 'fwd':
        x, Wk, b, s = R.fwd_operands(g, layer, 2, C, H, W, DEV)
        rc, y = _fwd(layer, x, Wk, b, s)
        return rc, [y], lambda: [R.forward(x, Wk, b, s, layer)]
    if kind == 'dw':
        x, dy, s = R.dw_operands(g, layer, 2, C, H, W, DEV)
        rc, sw, sb, guard = _dw(layer, x, dy, s, 3)
        return rc, [sw.double().sum(0), sb.double().sum(0), guard], lambda: [*R.weight_grad(x, dy, s, layer), None]
    dy, Wk, act = R.dx_operands(g, 2, C, H, W, DEV)
    rc, dx = _dx(dy, Wk, act, C, H, W)
    return rc, [dx], lambda: [R.input_grad(dy, Wk, act, C, H, W)]


@pytest.mark.parametrize('case', R.ENVELOPE_CASES, ids=['l%d_%s_%s_%d' % (c[0], c[1], c[5], c[6]) for c in R.ENVELOPE_CASES])
def test_envelope_edge(case):
    layer, kind, C, H, W, axis, top = case
    assert R.largest(layer, kind, C, H, W, axis) == top
    shape = lambda v: dict(C=(v, H, W), H=(C, v, W), W=(C, H, v), HW=(C, v, v))[axis]  # noqa: E731
    rc, outs, refs = _run(layer, kind, *shape(top), top)
    assert rc == OK, ('refused inside the envelope', case, R.envelope(layer, kind, *shape(top)))
    for got, ref in zip(outs, refs()):
        if ref is None:
            assert bool(torch.isnan(got).all())
        else:
            _exact(got, ref, ('envelope', case))
    rc, outs, _ = _run(layer, kind, *shape(top + 1), top + 1)
    assert rc == ERR_UNSUPPORTED, ('accepted past the envelope', case, rc)
    assert all(bool(torch.isnan(o).all()) for o in outs), 'a refused call wrote its output'


def test_forward_zero_frames_writes_nothing():
    for layer, C, H, W in ((1, 4, 84, 84), (2, 16, 20, 20)):
        x, Wk, b, s = R.fwd_operands(_gen(('zero', layer)), layer, 1, C, H, W, DEV)
        rc, y = _fwd(layer, x, Wk, b, s, frames=0)
        assert rc == OK and bool(torch.isnan(y).all())


@pytest.mark.parametrize('layer,kind,H,W', [(1, 'fwd', 7, 8), (1, 'fwd', 8, 7), (2, 'fwd', 3, 4), (1, 'dw', 7, 8),
                                            (1, 'dw', 8, 7), (2, 'dw', 3, 4), (2, 'dw', 4, 3), (2, 'dx', 3, 4),
                                            (2, 'dx', 4, 3)])
def test_frames_smaller_than_the_kernel_are_refused(layer, kind, H, W):
    """(H - KS) / ST truncates towards zero in C, so H = KS - 1 would compute one output row from a window that runs
    past the frame; every launch refuses it with SB200_ERR_ARG and writes nothing."""
    KS, _, CO = R.LAYERS[layer]
    C, n = (2, 2) if layer == 1 else (16, 2)
    x = torch.zeros(n, C, H, W, device=DEV)
    Wk = torch.zeros(C * KS * KS, CO, device=DEV)
    out = torch.full((n, C * H * W + CO * 4), NAN, device=DEV)
    dy = torch.zeros(n, CO, device=DEV)
    L, st = _lib_(), ops._stream()
    if kind == 'fwd':
        rc = L.sb200_conv_forward_f32(layer, _p(x), 0, n, C, H, W, _p(Wk), _p(Wk), 1.0, _p(out), st)
    elif kind == 'dw':
        rc = L.sb200_conv_backward_dw_f32(layer, _p(x), 0, _p(dy), n, C, H, W, 1.0, _p(out), _p(out), out.shape[1], 1, st)
    else:
        rc = L.sb200_conv_backward_dx_f32(2, _p(dy), _p(Wk), None, n, C, H, W, _p(out), st)
    torch.cuda.synchronize()
    assert rc == ERR_ARG and bool(torch.isnan(out).all())


# ---- d. one StemTrainer backward at the default pixel shapes -------------------------------------------------------
def test_stem_trainer_backward_default_shapes(rows):
    """CNNStem [4, 84, 84] -> 256 on M frames, StemTrainer.backward, the slabs reduced by sb200_grad_reduce_norm_f32.
    Each stage is compared with float64 autograd of Conv2d / Linear / ReLU on the fp32 tensors that stage read (the
    saved a1 / a2 and the kernels' d_a2 / d_a1): taken end to end, a pre-activation within rounding of 0 would flip a
    relu' mask and no bound would hold.  Convolutions: the bounded criterion with K = the slab chain + splits for the
    reduction.  Linear: test_grads_gpu.py's bars for the backward GEMMs, |g - g64| <= c |X|^T |dY| with c = 2e-7 (dW)
    and 1e-6 (dX)."""
    from surreal_b200.model.cnn_stem import CNNStem, StemTrainer
    M = rows['M']
    torch.manual_seed(11)
    stem = CNNStem((4, 84, 84), 256, DEV)
    tr = StemTrainer(stem, M)
    g = _gen('trainer')
    frames = torch.randint(0, 256, (M, 4, 84, 84), generator=g, device=DEV, dtype=torch.uint8)
    feat = tr.forward(frames)
    d_feat = torch.zeros(M, ops._ru(256, 4), device=DEV)
    d_feat[:, :256] = torch.randn(M, 256, generator=g, device=DEV) * (feat > 0)
    tr.backward(d_feat)
    L = _lib_()
    grad = torch.full((stem.size,), NAN, device=DEV)
    ws = torch.zeros(L.sb200_optim_workspace_bytes(), dtype=torch.uint8, device=DEV)
    _lib.check(L.sb200_grad_reduce_norm_f32(_p(tr.slabs), stem.size, tr.splits, _p(grad), stem.size, 1.0, 0, _p(ws), None,
                                            ops._stream()), 'reduce')
    torch.cuda.synchronize()
    a1, a2, sp = tr.bufs['a1'], tr.bufs['a2'], tr.splits
    seg = lambda name: stem.seg(name, grad)  # noqa: E731
    # Linear (flat -> 256) in the kernel layout [flat][ldw]
    lay = stem.fc.layout[0]
    o_fc = stem.off['fc'][0]
    Wfc = stem.params[o_fc + lay['w']:o_fc + lay['w'] + stem.flat * lay['ldw']].view(stem.flat, lay['ldw'])[:, :256].double()
    gfc_w = grad[o_fc + lay['w']:o_fc + lay['w'] + stem.flat * lay['ldw']].view(stem.flat, lay['ldw'])[:, :256].double()
    gfc_b = grad[o_fc + lay['b']:o_fc + lay['b'] + 256].double()
    X, dY = a2.double(), d_feat[:, :256].double()
    ratios = {'fc_w': float(((gfc_w - X.t() @ dY).abs() / (X.abs().t() @ dY.abs()).clamp_min(1e-300)).max()) / 2e-7,
              'fc_b': float(((gfc_b - dY.sum(0)).abs() / dY.abs().sum(0).clamp_min(1e-300)).max()) / 2e-7}
    ref_da2 = (dY @ Wfc.t()) * (X > 0)
    ratios['d_a2'] = float(((tr.d_a2.double() - ref_da2).abs() / (dY.abs() @ Wfc.abs().t()).clamp_min(1e-300)).max()) / 1e-6
    # conv2: dW from the saved a1 and the kernel's d_a2; d_a1 = dX masked by relu'(a1)
    d_a2 = tr.d_a2.view(M, 32, stem.H2, stem.W2)
    gw, gb = R.weight_grad(a1, d_a2, 1.0, 2)
    aw, ab = R.abs_weight_grad(a1, d_a2, 1.0, 2)
    K = R.chain_dw(2, M, sp, stem.H1, stem.W1) + sp
    ratios['conv2_w'] = _ratio(seg('w2').view(stem.taps2, 32), gw, aw, K)
    ratios['conv2_b'] = _ratio(seg('b2'), gb, ab, K)
    W2 = stem.seg('w2').view(stem.taps2, 32)
    ratios['d_a1'] = _ratio(tr.d_a1, R.input_grad(d_a2, W2, a1, 16, stem.H1, stem.W1),
                            R.abs_input_grad(d_a2, W2, 16, stem.H1, stem.W1), R.chain_dx())
    # conv1: dW from the frames / 255 and the kernel's d_a1
    gw, gb = R.weight_grad(frames, tr.d_a1, 1.0 / 255.0, 1)
    aw, ab = R.abs_weight_grad(frames, tr.d_a1, 1.0 / 255.0, 1)
    K = R.chain_dw(1, M, sp, 84, 84) + sp
    ratios['conv1_w'] = _ratio(seg('w1').view(stem.taps1, 16), gw, aw, K)
    ratios['conv1_b'] = _ratio(seg('b1'), gb, ab, K)
    print('measured trainer bound ratio', M, sp, ratios)
    assert all(r <= 1.0 for r in ratios.values()), ratios

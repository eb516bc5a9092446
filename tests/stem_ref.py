"""Float64 restatement of the CNN stem convolutions (csrc/stem.cu), their shared-memory envelope, and operand builders
whose fp32 arithmetic is exact.

The three operations as the kernels define them (Wk in the kernel layout [(c, ky, kx)][COUT], x multiplied by in_scale):
  forward  y  = relu(conv2d(x * in_scale, W, b, stride))
  dW / db  the weight / bias gradient of conv2d(x * in_scale) for dy = the gradient w.r.t. the PRE-activation
  dX       (layer 2) the input gradient of conv2d for that dy, times relu'(act) = (act > 0), or unmasked without act
Each has an ``abs_*`` twin: the same sums over |x|, |W|, |b|, |dy|, i.e. S = sum |terms| of every output, the scale of the
a-priori rounding bound  |fp32 - exact| <= gamma_K * S  of a K-long chain of fp32 multiply-adds.

Exact operands: frames are integers (uint8, in_scale = 2^-k), post-ReLU layer-2 inputs k/16, weights and biases k/64
with |k| <= 64, dy in {-1, 0, 1}.  Every term is then an integer multiple of one unit q, and while the sum of |terms| of
an output stays below 2^24 q every product and every partial sum, in any order, is an fp32 number: the kernel's result
equals the float64 one exactly.  Each builder asserts that condition from the shapes and value ranges it draws."""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24                 # fp32 unit roundoff
U64 = 2.0 ** -53
EXACT_LIMIT = 2 ** 24
SMEM_MAX = 200 * 1024          # STEM_SMEM_MAX: each launch refuses more dynamic shared memory than this
GRID_CAP = 132 * 4             # forward and dX launch min(frames, 528) CTAs and walk the frames grid-stride
LAYERS = {1: (8, 4, 16), 2: (4, 2, 32)}      # KS, ST, COUT


def out_hw(layer, H, W):
    KS, ST, _ = LAYERS[layer]
    return (H - KS) // ST + 1, (W - KS) // ST + 1


def to_torch(Wk, C, layer):
    """kernel layout [(c, ky, kx)][COUT] -> torch [COUT][C][KS][KS]"""
    KS, _, CO = LAYERS[layer]
    return Wk.reshape(C * KS * KS, CO).t().reshape(CO, C, KS, KS)


def to_kernel(w):
    """torch [COUT][C][KS][KS] -> kernel layout [(c, ky, kx)][COUT]"""
    return w.reshape(w.shape[0], -1).t().contiguous()


def _f64(t):
    return t.to(torch.float64)


def _no_cudnn():
    # cuDNN may pick FFT / Winograd algorithms, which round even integer data; the native convolution is im2col + GEMM
    return torch.backends.cudnn.flags(enabled=False)


# ---- float64 reference ---------------------------------------------------------------------------------------------
def forward(x, Wk, b, in_scale, layer):
    """y = relu(conv2d(x * in_scale, W, b)) in float64"""
    C = x.shape[1]
    with _no_cudnn():
        return torch.relu(F.conv2d(_f64(x) * in_scale, to_torch(_f64(Wk), C, layer), _f64(b), stride=LAYERS[layer][1]))


def abs_forward(x, Wk, b, in_scale, layer):
    C = x.shape[1]
    with _no_cudnn():
        return F.conv2d(_f64(x).abs() * abs(in_scale), to_torch(_f64(Wk).abs(), C, layer), _f64(b).abs(),
                        stride=LAYERS[layer][1])


def weight_grad(x, dy, in_scale, layer):
    """(dWk [taps][COUT], db [COUT]) of conv2d(x * in_scale) for the pre-activation gradient dy, by float64 autograd"""
    KS, ST, CO = LAYERS[layer]
    w = torch.zeros(CO, x.shape[1], KS, KS, dtype=torch.float64, device=x.device, requires_grad=True)
    b = torch.zeros(CO, dtype=torch.float64, device=x.device, requires_grad=True)
    with _no_cudnn():
        gw, gb = torch.autograd.grad(F.conv2d(_f64(x) * in_scale, w, b, stride=ST), (w, b), _f64(dy))
    return to_kernel(gw), gb


def abs_weight_grad(x, dy, in_scale, layer):
    return weight_grad(_f64(x).abs(), _f64(dy).abs(), abs(in_scale), layer)


def input_grad(dy, Wk, act, C, H, W, layer=2):
    """dX [frames][C][H][W] of conv2d for dy, times (act > 0) unless act is None, by float64 autograd"""
    KS, ST, _ = LAYERS[layer]
    x = torch.zeros(dy.shape[0], C, H, W, dtype=torch.float64, device=dy.device, requires_grad=True)
    with _no_cudnn():
        gx, = torch.autograd.grad(F.conv2d(x, to_torch(_f64(Wk), C, layer), stride=ST), (x,), _f64(dy))
    return gx if act is None else gx * (_f64(act) > 0)


def abs_input_grad(dy, Wk, C, H, W, layer=2):
    return input_grad(_f64(dy).abs(), _f64(Wk).abs(), None, C, H, W, layer)


# ---- chain lengths and the a-priori bound ---------------------------------------------------------------------------
def gamma(k, u=U):
    return k * u / (1.0 - k * u)


def chain_fwd(layer, C):
    """C * KS^2 multiply-adds into one accumulator, then the bias add"""
    KS = LAYERS[layer][0]
    return C * KS * KS + 1


def chain_dw(layer, frames, splits, H, W):
    """one CTA sums its ceil(frames / splits) frames x HO * WO positions into one accumulator per weight"""
    HO, WO = out_hw(layer, H, W)
    return -(-frames // splits) * HO * WO


def chain_dx(layer=2):
    """at most ceil(KS / ST)^2 taps x COUT channels reach one input pixel"""
    KS, ST, CO = LAYERS[layer]
    return (-(-KS // ST)) ** 2 * CO


def bound(S, K):
    """|fp32 result - float64 reference| for a K-long fp32 chain with sum |terms| = S.  The kernels take in_scale as an
    fp32 number and round x * in_scale: each input is x * in_scale * (1 + d1)(1 + d2), |d| <= u, which moves the exact
    sum by at most (2u + u^2) S; the chain over the rounded terms (sum |terms| <= (1 + u)^2 S) adds at most
    gamma_K (1 + u)^2 S <= gamma_{K+2} S.  The float64 reference adds at most gamma_{K+2}(2^-53) S of its own."""
    return (gamma(K + 2) + 2 * U + U * U + gamma(K + 2, U64)) * S


# ---- shared-memory envelope -----------------------------------------------------------------------------------------
def ru4(v):
    return (v + 3) & ~3


def row_pitch(layer, W):
    KS, ST, _ = LAYERS[layer]
    return ru4(W + 3 * ST + KS)


def envelope(layer, kind, C, H, W):
    """Dynamic shared memory in bytes of one launch: kind 'fwd' (launch_fwd), 'dw' (launch_dw) or 'dx'
    (sb200_conv_backward_dx_f32, layer 2 only)."""
    KS, ST, CO = LAYERS[layer]
    HO, WO = out_hw(layer, H, W)
    if kind == 'fwd':
        floats = C * KS * KS * CO + C * H * row_pitch(layer, W)
    elif kind == 'dw':
        floats = ru4(C * H * W) + HO * WO * CO
    else:
        assert kind == 'dx' and layer == 2
        floats = C * KS * KS * CO + HO * WO * CO
    return 4 * floats


def accepts(layer, kind, C, H, W):
    return envelope(layer, kind, C, H, W) <= SMEM_MAX


def largest(layer, kind, C, H, W, axis):
    """The largest value of ``axis`` ('C', 'H', 'W' or 'HW' for square frames) the launch accepts, the others held at
    (C, H, W).  Shared memory grows monotonically along every axis."""
    def shape(v):
        return dict(C=(v, H, W), H=(C, v, W), W=(C, H, v), HW=(C, v, v))[axis]
    v = dict(C=C, H=H, W=W, HW=H)[axis]
    assert accepts(layer, kind, *shape(v))
    while accepts(layer, kind, *shape(v + 1)):
        v += 1
    return v


# ---- exact operand builders -----------------------------------------------------------------------------------------
def _ints(gen, lo, hi, shape, device):
    return torch.randint(lo, hi + 1, shape, generator=gen, device=device)


def weights(gen, C, layer, device):
    """Wk [taps][COUT] and bias [COUT], k / 64 with |k| <= 64"""
    KS, _, CO = LAYERS[layer]
    return (_ints(gen, -64, 64, (C * KS * KS, CO), device).float() / 64,
            _ints(gen, -64, 64, (CO,), device).float() / 64)


def inputs(gen, layer, frames, C, H, W, device, xmax=255, fill=None, u8=None, in_scale=1.0):
    """(x, in_scale, q_x): layer 1 integer frames in [0, xmax] (uint8, or float with in_scale = 2^-k), layer 2 post-ReLU
    maps k / 16 with about a third exact zeros.  ``fill`` sets every value to it.  q_x is the unit of x * in_scale."""
    assert math.frexp(in_scale)[0] == 0.5 and in_scale <= 1.0, 'in_scale must be a power of two'
    shape = (frames, C, H, W)
    if fill is not None:
        k = torch.full(shape, int(fill), dtype=torch.int64, device=device)
    else:
        k = _ints(gen, 0, xmax, shape, device)
    if layer == 1:
        x = k.to(torch.uint8) if u8 is not False else k.float()
        return x, in_scale, in_scale
    assert not u8 and in_scale == 1.0
    if fill is None:
        k[torch.rand(shape, generator=gen, device=device) < 0.33] = 0
    return k.float() / 16, 1.0, 1.0 / 16


def fwd_operands(gen, layer, frames, C, H, W, device, xmax=255, **kw):
    """forward operands; asserts  C KS^2 max|x s| max|w| + max|b| < 2^24 q  with q = q_x / 64"""
    KS = LAYERS[layer][0]
    x, s, qx = inputs(gen, layer, frames, C, H, W, device, xmax=xmax, **kw)
    Wk, b = weights(gen, C, layer, device)
    xm = (kw['fill'] if kw.get('fill') is not None else xmax) * qx
    S, q = C * KS * KS * xm * 1.0 + 1.0, qx / 64
    assert S / q < EXACT_LIMIT, ('forward operands not exact in fp32', layer, C, xmax, S / q)
    return x, Wk, b, s


def dy_sparse(gen, frames, layer, H, W, nz, device):
    """dy [frames][COUT][HO][WO] in {-1, 0, 1} with exactly nz nonzeros per (frame, channel)"""
    _, _, CO = LAYERS[layer]
    HO, WO = out_hw(layer, H, W)
    npos = HO * WO
    assert 1 <= nz <= npos
    pick = torch.rand(frames, CO, npos, generator=gen, device=device).argsort(-1) < nz
    sign = _ints(gen, 0, 1, (frames, CO, npos), device).float() * 2 - 1
    return (pick.float() * sign).view(frames, CO, HO, WO)


def dw_nz(layer, frames, H, W, xmax):
    """the densest dy (nonzeros per frame and channel) whose dW sums stay exact: frames * nz * xmax < 2^24 (units q_x)"""
    HO, WO = out_hw(layer, H, W)
    return min(HO * WO, (EXACT_LIMIT - 1) // (frames * max(1, xmax)))


def dw_operands(gen, layer, frames, C, H, W, device, xmax=255, nz=None, **kw):
    """dW operands (x, dy, in_scale).  One weight sums x * s * dy over at most frames * nz (frame, position) pairs with
    dy != 0 -- every slab and the slab total; asserts  frames * nz * max|x| < 2^24 (units q_x) and frames * nz < 2^24
    (the bias)."""
    x, s, _ = inputs(gen, layer, frames, C, H, W, device, xmax=xmax, **kw)
    xm = kw['fill'] if kw.get('fill') is not None else xmax
    nz = dw_nz(layer, frames, H, W, xm) if nz is None else nz
    assert nz >= 1 and frames * nz * max(1, xm) < EXACT_LIMIT, ('dW operands not exact in fp32', layer, frames, nz, xm)
    return x, dy_sparse(gen, frames, layer, H, W, nz, device), s


def dx_operands(gen, frames, C, H, W, device):
    """dX operands (dy, Wk, act) of layer 2: dy in {-1, 0, 1}, Wk k / 64, act k / 16 >= 0 with about a third exact zeros;
    asserts  ceil(KS/ST)^2 COUT max|dy| max|w| < 2^24 q  with q = 1 / 64"""
    HO, WO = out_hw(2, H, W)
    dy = _ints(gen, -1, 1, (frames, LAYERS[2][2], HO, WO), device).float()
    Wk, _ = weights(gen, C, 2, device)
    act, _, _ = inputs(gen, 2, frames, C, H, W, device)
    assert chain_dx() * 1.0 * 1.0 * 64 < EXACT_LIMIT
    return dy, Wk, act


# ---- the shapes the GPU tests run ------------------------------------------------------------------------------------
# frames 'M' / 'ALL': the default-config pixel PPOLearner's update rows B * eff_len and critic rows B * (n + 1);
# splits 'trainer': StemTrainer's choice max(1, min(16, frames // 16)).  Each id names the kernel path it covers.
_L1, _L2 = (4, 84, 84), (16, 20, 20)
FWD_CASES = [
    ('learner_M_l1', 1, 'M', *_L1, {}), ('learner_ALL_l1', 1, 'ALL', *_L1, {}),
    ('learner_M_l2', 2, 'M', *_L2, {}), ('learner_ALL_l2', 2, 'ALL', *_L2, {}),
] + [('grid_stride_frames%d_l%d' % (n, layer), layer, n, *shape, {})
     for n in (1, 527, 528, 529, 1057) for layer, shape in ((1, (2, 20, 28)), (2, (16, 9, 11)))] + [
    ('masked_col_group_wo%d_l1' % wo, 1, 3, 3, 12, 4 * wo + 4, {}) for wo in (4, 5, 6, 7)] + [
    ('masked_col_group_wo%d_l2' % wo, 2, 3, 16, 6, 2 * wo + 2, {}) for wo in (4, 5, 6, 7)] + [
    ('ho1_l1', 1, 4, 3, 8, 36, {}), ('wo1_l1', 1, 4, 3, 36, 8, {}), ('ho1_wo1_l1', 1, 4, 3, 8, 8, {}),
    ('ho1_l2', 2, 4, 16, 4, 13, {}), ('wo1_l2', 2, 4, 16, 13, 4, {}), ('ho1_wo1_l2', 2, 4, 16, 4, 4, {}),
    ('nonsquare_l1', 1, 5, 3, 52, 100, {}), ('nonsquare_l2', 2, 5, 16, 21, 8, {}),
    ('u8_all0', 1, 3, *_L1, dict(fill=0)), ('u8_all255', 1, 3, *_L1, dict(fill=255)),
    ('u8_scale_2^-3', 1, 3, *_L1, dict(in_scale=0.125)),
    ('float_input_l1', 1, 5, 3, 33, 45, dict(u8=False, in_scale=0.25)),
    ('c5_l1', 1, 3, 5, 84, 84, {}), ('c17_l2', 2, 3, 17, 10, 10, {}),
]
DW_CASES = [
    ('learner_M_l1', 1, 'M', *_L1, 'trainer', {}), ('learner_ALL_l1', 1, 'ALL', *_L1, 'trainer', {}),
    ('learner_M_l2', 2, 'M', *_L2, 'trainer', {}), ('learner_ALL_l2', 2, 'ALL', *_L2, 'trainer', {}),
] + [('splits%d_l%d' % (s, layer), layer, 37, *shape, s, {})
     for s in (1, 7, 16) for layer, shape in ((1, (3, 28, 36)), (2, (16, 9, 11)))] + [
    ('idle_slabs_5of16_l1', 1, 5, 2, 20, 20, 16, {}), ('idle_slabs_1of7_l2', 2, 1, 16, 9, 9, 7, {}),
    ('frames1057_l2', 2, 1057, 16, 9, 11, 16, {}),
    ('tap_batch2_c5_l1', 1, 9, 5, 84, 84, 4, {}), ('tap_batch2_c17_l2', 2, 9, 17, 10, 10, 4, {}),
    ('ho1_l1', 1, 6, 2, 8, 30, 3, {}), ('wo1_l2', 2, 6, 16, 11, 4, 3, {}), ('ho1_wo1_l2', 2, 6, 16, 4, 4, 3, {}),
    ('nonsquare_l1', 1, 6, 3, 52, 100, 3, {}),
    ('u8_all0', 1, 4, *_L1, 2, dict(fill=0)), ('u8_all255', 1, 4, *_L1, 2, dict(fill=255)),
    ('float_input_l1', 1, 7, 3, 33, 45, 3, dict(u8=False, in_scale=0.25)),
]
DX_CASES = [('learner_M', 'M', *_L2), ('learner_ALL', 'ALL', *_L2)] + [
    ('grid_stride_frames%d' % n, n, 16, 9, 11) for n in (1, 527, 528, 529, 1057)] + [
    ('ho1_wo1', 4, 16, 4, 4), ('ho1', 4, 16, 4, 13), ('wo1', 4, 16, 13, 4), ('nonsquare_c5', 6, 5, 15, 22)]
# (layer, kind, C, H, W, axis, the largest accepted value along axis): the launches' shared-memory envelope
ENVELOPE_CASES = [
    (1, 'fwd', *_L1, 'C', 5), (1, 'fwd', *_L1, 'H', 113), (1, 'fwd', *_L1, 'W', 120),
    (1, 'fwd', 1, 84, 84, 'HW', 212), (1, 'fwd', 4, 84, 84, 'HW', 98),
    (2, 'fwd', *_L2, 'C', 44), (2, 'fwd', *_L2, 'H', 84), (2, 'fwd', *_L2, 'W', 122),
    (1, 'dw', *_L1, 'C', 6), (1, 'dw', *_L1, 'H', 123), (1, 'dw', *_L1, 'W', 123),
    (1, 'dw', 1, 84, 84, 'HW', 163), (1, 'dw', 4, 84, 84, 'HW', 102),
    (2, 'dw', *_L2, 'C', 121), (2, 'dw', *_L2, 'H', 111), (2, 'dw', *_L2, 'W', 111),
    (2, 'dx', *_L2, 'C', 94), (2, 'dx', *_L2, 'H', 301), (2, 'dx', *_L2, 'W', 301),
]


def learner_rows(B, n_step, horizon):
    """(M, ALL) of a recurrent pixel PPOLearner: B * (n - horizon + 1) update rows, B * (n + 1) critic rows"""
    return B * (n_step - horizon + 1), B * (n_step + 1)


def resolve(frames, splits, rows):
    n = rows[frames] if isinstance(frames, str) else frames
    return n, (max(1, min(16, n // 16)) if splits == 'trainer' else splits)

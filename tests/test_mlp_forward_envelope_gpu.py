"""Every fused-MLP forward kernel against float64 across the dispatch envelope of mlp_forward_impl (mlp_fwd.cu): the
skinny kernel, the 3xTF32 mma.sync tiles, each FFMA tile instantiation, the wgmma kernel (Tc5Forward) and the packed
cluster kernel (PackedWeights), at the row, width, head and z-filter edges where each family changes behaviour.

Each case names the kernel family it is meant to reach, and the CUDA activity trace (torch.profiler) must show that
kernel: a change to a dispatch threshold that moves a case to another family fails here instead of silently dropping
the coverage.  The widths and row counts are derived below from the same shared-memory plans the dispatcher uses.

Numerics, per layer l on the kernel's own float32 input h (the saved output of layer l-1, or save_x):
    |y - act(h @ W^T + b)_64| <= c * (|h| @ |W|^T + |b|)        element-wise, exact where the right side is 0,
plus 4 ulp of |y| after a tanh (tanhf).  ReLU and tanh are 1-Lipschitz, so the bound on the pre-activation holds after
them.  The wgmma and packed kernels write only their output; there the same bound is carried through the layers in
float64 (the rounding of layer l enters layer l+1 through |W|), a looser bound whose c is on its own scale.  One c per
family; measured worst over this file on an H100 SXM (700 W), and the bar:

    skinny  mlp_fwd_skinny_kernel    2.7e-7  1e-6      t2_64   mlp_fwd_kernel<2, 64>    3.1e-7  1e-6
    mma1    mlp_fwd_mma_kernel<1>    1.8e-6  4e-6      t2_16   mlp_fwd_kernel<2, 16>    3.2e-7  1e-6
    mma2    mlp_fwd_mma_kernel<2>    1.4e-6  4e-6      t1_64   mlp_fwd_kernel<1, 64>    2.3e-7  1e-6
    t8_16   mlp_fwd_kernel<8, 16>    3.7e-7  1e-6      t1_16   mlp_fwd_kernel<1, 16>    3.3e-7  1e-6
    t4_16   mlp_fwd_kernel<4, 16>    3.4e-7  1e-6      tc5     mlp3_wgmma_kernel        7.8e-9  5e-8  (carried bound)
                                                       pk      mlp_fwd_pk_kernel        1.2e-8  5e-8  (carried bound)

Plain single-pass TF32 products (the 3xTF32 correction terms dropped) measure ~4e-4 in the per-layer bound and ~9e-7 in
the carried one.
"""
import os
import subprocess
import sys

import pytest
import torch

from surreal_b200 import _lib, ops

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
U = 2.0 ** -24                  # float32 unit roundoff
EPS = 1e-5                      # z-filter std floor (ZFilter's eps)
RELU, TANH, NONE = ops.ACT_RELU, ops.ACT_TANH, ops.ACT_NONE
PADR = 3                        # extra rows past every output, save and save_x buffer: must stay NaN

KERNEL = {
    'skinny': 'mlp_fwd_skinny_kernel',
    'mma1': 'mlp_fwd_mma_kernel<1>',
    'mma2': 'mlp_fwd_mma_kernel<2>',
    't8_16': 'mlp_fwd_kernel<8, 16>',
    't4_16': 'mlp_fwd_kernel<4, 16>',
    't2_64': 'mlp_fwd_kernel<2, 64>',
    't2_16': 'mlp_fwd_kernel<2, 16>',
    't1_64': 'mlp_fwd_kernel<1, 64>',
    't1_16': 'mlp_fwd_kernel<1, 16>',
    'tc5': 'mlp3_wgmma_kernel',
    'pk': 'mlp_fwd_pk_kernel',
}

# c per family: FFMA kernels accumulate in fp32 FMA chains; the tensor-core kernels drop the lo*lo term of the 3xTF32
# split (~2^-22 of |a||b| per product) and round the other two products to tf32 inputs.
C_BAR = {
    'skinny': 1e-6, 't8_16': 1e-6, 't4_16': 1e-6, 't2_64': 1e-6, 't2_16': 1e-6, 't1_64': 1e-6, 't1_16': 1e-6,
    'mma1': 4e-6, 'mma2': 4e-6, 'tc5': 5e-8, 'pk': 5e-8,
}

# ---- the dispatch plans of mlp_forward_impl / launch_fwd_mma (floats of dynamic shared memory) ---------------------
BUDGET = 200 * 1024 // 4            # SMEM_BUDGET: tile and mma kernels
SKINNY_BUDGET = 100 * 1024 // 4


def _ru(v, m):
    return (v + m - 1) // m * m


def _tile_fits(w, bm, bk):          # mlp_forward_impl's fits(bm, bk): two activation tiles + two BK x 256 weight stages
    return 2 * bm * (_ru(w, bk) + 4) + 2 * bk * 256 <= BUDGET


def _mma_fits(w, mt, scratch):      # launch_fwd_mma<MT>
    return 2 * 16 * mt * (_ru(w, 8) + 4) + scratch <= BUDGET


def _skinny_fits(w, scratch):
    return 2 * 8 * (_ru(w, 32) + 4) + scratch <= SKINNY_BUDGET


def _widest(pred):
    return max(w for w in range(1, 4097) if pred(w))


SCR = 32                            # scratch of the [16, W, 40] nets below: 2 * dims[0] floats, no narrow layer
W_T8 = _widest(lambda w: _tile_fits(w, 64, 16))          # 320
W_T4 = _widest(lambda w: _tile_fits(w, 32, 16))          # 656
W_T2_64 = _widest(lambda w: _tile_fits(w, 16, 64))       # 512
W_T2_16 = _widest(lambda w: _tile_fits(w, 16, 16))       # 1328
W_MAX = _widest(lambda w: _tile_fits(w, 8, 16))          # 2672: wider is SB200_ERR_ARG
W_SKINNY = _widest(lambda w: _skinny_fits(w, SCR))       # 1568
W_MMA1 = _widest(lambda w: _mma_fits(w, 1, SCR))         # 1592
W_MMA2 = _widest(lambda w: _mma_fits(w, 2, SCR))         # 792
# rows: skinny up to 2048 (8-row CTAs); mma<1> up to 4096, mma<2> above; in forward mode 0 the FFMA tiles take
# <4,16> from 240 32-row tiles, <8,16> from 120 64-row tiles, <4,16> from 120 32-row tiles, else <2,64> (want = 120)
R_T4_FROM = 119 * 32 + 1            # 3809
R_T8_FROM = 119 * 64 + 1            # 7617
R_T8_TO = 239 * 32                  # 7648


# ---- helpers -------------------------------------------------------------------------------------------------------
def _net(dims, acts=None, aux=None, seed=0, bscale=1.0):
    al, ad = aux if aux else (-1, 0)
    acts = acts or [RELU] * (len(dims) - 2) + [TANH if dims[-1] > 1 else NONE]
    net = ops.FlatNet(dims, acts, DEV, aux_layer=al, aux_dim=ad)
    g = torch.Generator(device=DEV).manual_seed(1000 + seed)
    for l, lay in enumerate(net.layout):
        K, N = lay['K'], lay['N']
        w = (torch.rand(N, K, generator=g, device=DEV) * 2 - 1) * K ** -0.5
        b = (torch.rand(N, generator=g, device=DEV) * 2 - 1) * K ** -0.5 * bscale
        b[::5] = 0.0                                    # with the zero rows of x: elements whose bound is exactly 0
        net.set_layer(l, w, b)
    return net


def _stats(kind, K0, g):
    """z-filter statistics [sum | sumsq | count] (float32).  'rand': 200 samples; 'init': ZFilter's initial state
    (sum 0, sumsq eps, count eps: mean 0, std 1); 'edge': count 64 and, in columns 0-3, a variance below eps^2, a
    variance of exactly 0 at mean 0.75, a negative variance (sumsq/count < mean^2 in float32 as in float64: sqrtf gives
    NaN, and fmaxf(NaN, eps) gives eps) and a std of 0.05 that clamps most values at +-5."""
    if kind == 'init':
        return torch.cat([torch.zeros(K0), torch.full((K0,), EPS), torch.tensor([EPS])]).to(DEV)
    n = 200 if kind == 'rand' else 64
    s = torch.randn(n, K0, generator=g, device=DEV, dtype=torch.float64) * 1.7 + 0.4
    st = torch.cat([s.sum(0), (s * s).sum(0), torch.tensor([float(n)], device=DEV, dtype=torch.float64)])
    if kind == 'edge':
        assert K0 >= 4
        for k, (sm, sq) in enumerate([(0.0, 64e-12), (48.0, 36.0), (64000.0, 64e6 * (1 - 1e-5)), (0.0, 0.16)]):
            st[k], st[K0 + k] = sm, sq
    return st.float()


def _edge_x(x, g):
    """Columns 0-3 for the 'edge' statistics: within +-4.8 of the floored std (eps) around the mean in columns 0 and 1,
    so that the floor shows in unclamped values; 1000 + {0, +-1, +-2} ulp in column 2 (z = 0 or clamped)."""
    n = x.shape[0]
    j = torch.randint(-12, 13, (n, 2), generator=g, device=DEV).float()
    x[:, 0] = j[:, 0] * 4e-6
    x[:, 1] = 0.75 + j[:, 1] * 4e-6
    x[:, 2] = 1000.0 + torch.randint(-2, 3, (n,), generator=g, device=DEV).float() * 2.0 ** -14
    return x


def _rnd32(v):
    """|fl32(v) - v|: the rounding of one IEEE float32 operation whose exact result is v (plus a float64 ulp)."""
    return (v.float().double() - v).abs() + 2.0 ** -52 * v.abs()


def _zfilter64(x64, stats, recip=False):
    """float64 z-filter: mean = sum / count, var = sumsq / count - mean^2, std = max(sqrt(var), eps) (eps where var < 0:
    the kernels' fmaxf(sqrtf(var), eps) maps the NaN to eps), z = clamp((x - mean) / std, -5, 5); and a bound on the
    float32 filter's rounding: one correctly rounded float32 operation each for the two quotients, mean^2 (0 if fused),
    the difference, sqrt, x - mean and the division (the clamp and the floor are 1-Lipschitz).  ``recip``: the filter
    multiplies by a rounded reciprocal of std (the wgmma kernel), one more rounding of z."""
    K0 = x64.shape[1]
    s = stats.double()
    cnt = s[2 * K0]
    mean, msq = s[:K0] / cnt, s[K0:2 * K0] / cnt
    var = msq - mean * mean
    e_m = _rnd32(mean)
    m32 = mean.float().double()
    e_var = _rnd32(msq) + 2 * mean.abs() * e_m + e_m * e_m + _rnd32(m32 * m32)
    e_var = e_var + U * (var.abs() + e_var)
    neg = var + e_var < 0                               # negative in float32 as in float64: NaN from sqrtf -> eps
    a = var.clamp(min=0).sqrt()
    e_a = torch.minimum(e_var.sqrt(), e_var / a.clamp(min=1e-300)) + U * (a + e_var.sqrt())
    std = torch.where(neg, torch.full_like(a, EPS), a.clamp(min=EPS))
    e_std = torch.where(neg | (a + e_a <= EPS), torch.zeros_like(a), e_a)   # floored on both sides: exactly eps
    d = x64 - mean
    zr = d / std
    e_z = (e_m + U * (d.abs() + e_m)) / std + zr.abs() * (e_std / std + (2 if recip else 1) * U)
    return zr.clamp(-5.0, 5.0), 1.5 * e_z + 1e-30


def _act64(h, act):
    return torch.relu(h) if act == RELU else (torch.tanh(h) if act == TANH else h)


def _check_writes(buf, rows, cols, what):
    """Every valid element written (finite), every padding element untouched (still NaN)."""
    assert bool(torch.isfinite(buf[:rows, :cols]).all()), '%s: a valid element is not finite (missed write?)' % what
    pad = torch.ones_like(buf, dtype=torch.bool)
    pad[:rows, :cols] = False
    assert bool(torch.isnan(buf[pad]).all()), '%s: a write outside [rows) x [cols)' % what


def _forward_kernels(fn, launches=True):
    """Run fn under the CUDA activity trace; the forward kernels it launched (demangled names).  The trace of this
    process now and then lacks kernel records of the library (seen on H100 hosts, a few cases in a few hundred): a
    library kernel launched after fn (sb200_add_f32) marks a complete trace, and a trace without the marker, or without
    any forward kernel where ``launches`` expects one, is taken again (fn writes the same values to the same places)."""
    mark = torch.zeros(1, device=DEV)
    for _ in range(5):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            _lib.check(_lib.lib().sb200_add_f32(mark.data_ptr(), mark.data_ptr(), 1, ops._stream()), 'sb200_add_f32')
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()}
        fwd = sorted(n for n in names if 'mlp_fwd' in n or 'mlp3_wgmma' in n)
        if any('add_kernel' in n for n in names) and (fwd or not launches):
            return fwd
    raise AssertionError('no complete CUDA activity trace in 5 runs; the last: %s' % sorted(names))


def _assert_family(names, family, what):
    if family is None:
        assert names == [], '%s: expected no launch, got %s' % (what, names)
        return
    assert len(names) == 1 and KERNEL[family] in names[0], \
        '%s: expected %s, the trace shows %s' % (what, KERNEL[family], names)


def _check_layers(net, h, aux64, ys, c, what):
    """The per-layer bound on the kernel's own inputs; returns the measured worst c."""
    worst = 0.0
    for l in range(net.n_layers):
        if net.aux_layer == l:
            h = torch.cat([h, aux64], 1)
        w, b = (t.double() for t in net.get_layer(l))
        ref = _act64(torch.addmm(b, h, w.t()), net.acts[l])
        scale = torch.addmm(b.abs(), h.abs(), w.abs().t())
        y = ys[l].double()
        err = (y - ref).abs()
        slack = 4 * U * y.abs() if net.acts[l] == TANH else torch.zeros_like(y)
        zero = scale == 0
        assert torch.equal(y[zero], ref[zero]), '%s layer %d: inexact where the bound is 0' % (what, l)
        r = float(((err - slack).clamp(min=0) / scale.masked_fill(zero, 1.0)).max()) if y.numel() else 0.0
        worst = max(worst, r)
        assert r <= c, '%s layer %d: |y - y64| reaches %.3g x (|h||W| + |b|) > c = %.3g' % (what, l, r, c)
        h = y
    return worst


def _check_chain(net, h, e0, aux64, out, c, what):
    """Output-only kernels: the per-layer bound carried through the net in float64.  err <= c * A + B, A the rounding
    of every layer propagated through |W|, B the z-filter's rounding (and tanhf's) propagated the same way."""
    A = torch.zeros_like(h)
    B = e0
    for l in range(net.n_layers):
        if net.aux_layer == l:
            h = torch.cat([h, aux64], 1)
            A = torch.cat([A, torch.zeros_like(aux64)], 1)
            B = torch.cat([B, torch.zeros_like(aux64)], 1)
        w, b = (t.double() for t in net.get_layer(l))
        aw = w.abs().t()
        A = torch.addmm(b.abs(), h.abs(), aw) + A @ aw
        B = B @ aw
        h = _act64(torch.addmm(b, h, w.t()), net.acts[l])
        if net.acts[l] == TANH:
            B = B + 4 * U * h.abs()
    err = (out.double() - h).abs()
    zero = (A == 0) & (B == 0)
    assert torch.equal(err[zero], torch.zeros_like(err[zero])), '%s: inexact where the bound is 0' % what
    r = float((err / (A + B / c)).masked_fill(zero, 0.0).max())      # r <= c: err <= c * A + B
    assert r <= c, '%s: |y - y64| reaches %.3g x (A + B / c) > c = %.3g' % (what, r, c)
    return r


def _set_mode(mode):
    _lib.check(_lib.lib().sb200_set_forward_mode(int(mode)), 'sb200_set_forward_mode')


# ---- the dispatched forward (sb200_mlp_forward_f32 / _variant_f32) ------------------------------------------------
def _run_case(case):
    """Run one case: every layer saved, save_x, NaN-filled padded buffers; assert the family, the writes, the z-filter
    and the per-layer bound.  Returns the launched kernel names."""
    ops._stream()
    dims, rows, family = case['dims'], case['rows'], case['family']
    zf, layout, padc = case.get('zf'), case.get('layout', 'plain'), case.get('padc', 4)
    what = case['id']
    net = _net(dims, case.get('acts'), case.get('aux'), seed=len(what) + rows, bscale=case.get('scale', 1.0))
    g = torch.Generator(device=DEV).manual_seed(rows + sum(dims))
    D, n = dims[0], max(rows, 1)
    x = torch.randn(n, D, generator=g, device=DEV) * 2 + 0.5
    if zf is None:
        x[::11] = 0.0
    if zf == 'edge':
        x = _edge_x(x, g)
    x = x * case.get('scale', 1.0)
    stats = _stats(zf, D, g) if zf else None
    kw = dict(zf_stats=stats, zf_eps=EPS, variant=case.get('variant', 0))
    if layout == 'window':
        wn = case.get('win_n', 3)
        assert rows % (wn + 1) == 0
        x3 = x.view(rows // (wn + 1), wn + 1, D)
        xarg = x3[:, :wn].contiguous()
        kw.update(x_next=x3[:, wn:].contiguous(), win_n=wn)
    elif layout == 'strided':
        ldx = 3 * D + 1
        xarg = torch.full((n, ldx), float('nan'), device=DEV)
        xarg[:, :D] = x
        kw.update(rows=rows, ldx=ldx)
    else:
        xarg = x
        kw.update(rows=rows, ldx=D)
    aux64 = None
    if case.get('aux'):
        ad = case['aux'][1]
        abuf = torch.full((n, ad + 3), float('nan'), device=DEV)
        abuf[:, :ad] = torch.rand(n, ad, generator=g, device=DEV) * 2 - 1
        kw['aux'] = abuf[:, :ad]
        aux64 = abuf[:rows, :ad].double()
    bufs = [torch.full((rows + PADR, N + padc), float('nan'), device=DEV) for N in dims[1:]]
    sxb = torch.full((rows + PADR, D + padc), float('nan'), device=DEV)
    kw['saves'] = [bb[:rows, :N] for bb, N in zip(bufs, dims[1:])]
    kw['save_x'] = sxb[:rows, :D]
    _set_mode(case.get('mode', 1))
    try:
        names = _forward_kernels(lambda: ops.mlp_forward(net, xarg, **kw), launches=family is not None)
    finally:
        _set_mode(1)
    _assert_family(names, family, what)
    for l, (bb, N) in enumerate(zip(bufs, dims[1:])):
        _check_writes(bb, rows, N, '%s save %d' % (what, l))
    _check_writes(sxb, rows, D, '%s save_x' % what)
    if rows == 0:
        return names
    x64, sx = x[:rows].double(), sxb[:rows, :D].double()
    if zf:
        z, ez = _zfilter64(x64, stats)
        zr = float(((sx - z).abs() / ez.clamp(min=1e-300)).max())
        assert bool(((sx - z).abs() <= ez).all()), '%s: save_x off the float64 filter: %.3g x its bound' % (what, zr)
        if zf == 'edge':      # the floored std shows in unclamped values; most of column 3 clamps
            assert rows < 9 or float(z[:, :2].abs().max()) > 3.0
            assert rows < 9 or float((sx[:, 3].abs() == 5.0).double().mean()) > 0.8
    else:
        assert torch.equal(sx, x64), '%s: save_x without a filter must be x' % what
    worst = _check_layers(net, sx, aux64, [bb[:rows, :N] for bb, N in zip(bufs, dims[1:])], C_BAR[family], what)
    print('measured %s %s c=%.3e' % (family, what, worst))
    return names


# the families the layer, head and layout features run on: (label, family, forward mode, variant, rows)
FAMILIES = [
    ('skinny', 'skinny', 1, 0, 37),
    ('mma1', 'mma1', 1, 0, 2100),
    ('mma2', 'mma2', 1, 0, 4500),
    ('mma2v1', 'mma2', 1, 1, 333),
    ('t2_64', 't2_64', 0, 0, 2100),
    ('t4_16v2', 't4_16', 1, 2, 333),
    ('t8_16', 't8_16', 0, 0, 7620),
]
FEATURES = [
    ('l1-narrow', dict(dims=[24, 5], zf='rand')),
    ('l1-wide', dict(dims=[24, 300])),
    ('l4', dict(dims=[20, 64, 48, 40, 6], zf='rand')),
    ('tanh-none-hidden', dict(dims=[20, 64, 48, 6], acts=[TANH, NONE, TANH])),
    ('k1', dict(dims=[1, 64, 40, 3])),
    ('k3', dict(dims=[3, 40, 3], zf='init')),
    ('k5', dict(dims=[5, 72, 33, 1], zf='rand')),
    ('aux0', dict(dims=[10, 64, 8], aux=(0, 3))),
    ('aux1', dict(dims=[10, 64, 40, 8], aux=(1, 5), zf='rand')),
    ('aux2-head', dict(dims=[10, 64, 48, 8], aux=(2, 6))),
    ('aux2-wide', dict(dims=[10, 64, 48, 40, 8], aux=(2, 6))),
    ('strided', dict(dims=[13, 200, 72, 6], layout='strided', zf='rand')),
    ('window', dict(dims=[13, 200, 72, 1], layout='window', zf='rand')),
    ('window-nozf', dict(dims=[13, 100, 1], layout='window')),
    ('act1e-3', dict(dims=[64, 256, 256, 8], scale=1e-3)),
    ('zf-edge', dict(dims=[12, 96, 64, 4], zf='edge')),
    ('zf-init', dict(dims=[12, 96, 64, 4], zf='init')),
    ('odd-ld', dict(dims=[17, 300, 200, 6], zf='rand', padc=3)),
] + [('head%d' % N, dict(dims=[16, 96, 64, N], zf='rand')) for N in (1, 8, 31, 32, 33, 300)]

CASES = []
for _lab, _fam, _mode, _var, _rows in FAMILIES:
    for _feat, _o in FEATURES:
        _r = _rows - _rows % 4 if _o.get('layout') == 'window' else _rows
        CASES.append(dict(_o, id='%s-%s' % (_lab, _feat), family=_fam, mode=_mode, variant=_var, rows=_r))

# rows at the family and tile edges ([13, 200, 72, 6]: every family's default shape)
for _mode, _rows, _fam in [(1, 0, None), (1, 1, 'skinny'), (1, 7, 'skinny'), (1, 8, 'skinny'), (1, 9, 'skinny'),
                           (1, 2048, 'skinny'), (1, 2049, 'mma1'), (1, 4096, 'mma1'), (1, 4097, 'mma2'),
                           (1, 50001, 'mma2'), (0, 9, 'skinny'), (0, 2049, 't2_64'), (0, R_T4_FROM - 1, 't2_64'),
                           (0, R_T4_FROM, 't4_16'), (0, R_T8_FROM - 1, 't4_16'), (0, R_T8_FROM, 't8_16'),
                           (0, R_T8_TO, 't8_16'), (0, R_T8_TO + 1, 't4_16'), (0, 50001, 't4_16')]:
    CASES.append(dict(id='rows%d-mode%d' % (_rows, _mode), family=_fam, mode=_mode, rows=_rows, dims=[13, 200, 72, 6],
                      zf='rand', padc=3))

# the widest layer on each side of every fit limit ([16, W, 40]: W is the widest layer input)
for _w, _mode, _rows, _fam in [(W_T8, 0, R_T8_FROM, 't8_16'), (W_T8 + 1, 0, R_T8_FROM, 't4_16'),
                               (W_T2_64, 0, 3000, 't2_64'), (W_T2_64 + 1, 0, 3000, 't2_16'),
                               (W_T4, 0, 4000, 't4_16'), (W_T4 + 1, 0, 4000, 't2_16'),
                               (W_MMA2, 1, 4097, 'mma2'), (W_MMA2 + 1, 1, 4097, 't2_16'),
                               (W_T2_16, 0, 3000, 't2_16'), (W_T2_16 + 1, 0, 3000, 't1_16'),
                               (W_SKINNY, 1, 2048, 'skinny'), (W_SKINNY + 1, 1, 2048, 't1_16'),
                               (W_MMA1, 1, 2049, 'mma1'), (W_MMA1 + 1, 1, 2049, 't1_16'),
                               (W_MAX, 1, 37, 't1_16')]:
    CASES.append(dict(id='w%d-mode%d-rows%d' % (_w, _mode, _rows), family=_fam, mode=_mode, rows=_rows,
                      dims=[16, _w, 40], zf='rand', padc=3))

# a narrow head with K * ldw on each side of the shared-memory staging limit: 16384 floats for the skinny and mma
# kernels, 2 * BK * 256 for the FFMA tiles (8192 at BK = 16; at BK = 64 the <= 512-wide layers always fit 32768)
for _k, _n, _lab, _fam, _mode, _var, _rows in [
        (512, 32, 'skinny', 'skinny', 1, 0, 37), (513, 32, 'skinny', 'skinny', 1, 0, 37),
        (512, 32, 'mma1', 'mma1', 1, 0, 2100), (513, 32, 'mma1', 'mma1', 1, 0, 2100),
        (512, 32, 'mma2', 'mma2', 1, 0, 4500), (513, 32, 'mma2', 'mma2', 1, 0, 4500),
        (256, 32, 't4_16v2', 't4_16', 1, 2, 333), (257, 32, 't4_16v2', 't4_16', 1, 2, 333),
        (256, 32, 't8_16', 't8_16', 0, 0, 7620), (257, 32, 't8_16', 't8_16', 0, 0, 7620),
        (1024, 8, 't2_16', 't2_16', 0, 0, 3000), (1025, 8, 't2_16', 't2_16', 0, 0, 3000)]:
    CASES.append(dict(id='%s-head-k%d-n%d' % (_lab, _k, _n), family=_fam, mode=_mode, variant=_var, rows=_rows,
                      dims=[16, _k, _n], zf='rand'))


@pytest.mark.parametrize('case', CASES, ids=[c['id'] for c in CASES])
def test_forward_matches_float64(case):
    _run_case(case)


def test_over_wide_rejected_before_launch():
    """The widest layer fits(8, 16) accepts runs (t1_16 in the table above); one column more is SB200_ERR_ARG from the
    argument check, and no kernel is launched."""
    net = _net([16, W_MAX + 1, 40])
    x = torch.randn(37, 16, device=DEV)

    def call():
        with pytest.raises(_lib.SB200Error, match=r'\(status -1\)'):
            ops.mlp_forward(net, x)
    assert _forward_kernels(call, launches=False) == []


def test_mma4_is_unreachable():
    """mlp_forward_impl tries mlp_fwd_mma_kernel<4> only after mlp_fwd_mma_kernel<2> returned SB200_ERR_UNSUPPORTED,
    and <4> needs 2 * 64 * ldh + scratch floats where <2> needs 2 * 32 * ldh + scratch (same ldh and scratch): it never
    fits when <2> does not, so no input reaches it.  Just past the <2> limit, with and without a staged narrow head, the
    dispatch falls through to the FFMA tiles."""
    w_head = _widest(lambda w: _mma_fits(w, 2, max(2 * w, 48 * 32)))
    for dims in ([16, W_MMA2 + 1, 40], [w_head + 1, 48, 32]):
        names = _run_case(dict(id='past-mma2-%s' % dims, family='t2_16', mode=1, rows=4097, dims=dims, zf='rand'))
        assert not any('mlp_fwd_mma_kernel<4>' in n for n in names)
    for w in range(1, W_MAX + 1):
        for scratch in (2 * 16, 2 * w, 16384):
            assert _mma_fits(w, 2, scratch) or not _mma_fits(w, 4, scratch)


# ---- the wgmma kernel (Tc5Forward) ---------------------------------------------------------------------------------
TC5_CASES = [
    dict(id='k0max', dims=[256, 256, 256, 1], rows=1000, zf='rand'),
    dict(id='n1-lt-n2', dims=[64, 128, 256, 3], rows=777, zf='rand'),
    dict(id='n1-gt-n2-edge', dims=[32, 256, 64, 8], rows=3000, zf='edge'),
    dict(id='n1-partial-half', dims=[96, 160, 96, 4], rows=128, zf='init'),
    dict(id='nout2', dims=[64, 256, 256, 2], rows=129),
    dict(id='nout5', dims=[64, 256, 256, 5], rows=1000, zf='rand'),
    dict(id='nout7', dims=[64, 256, 256, 7], rows=640),
    dict(id='window', dims=[64, 256, 256, 1], rows=150 * 17, win_n=16, zf='rand'),
    dict(id='grid3', dims=[64, 256, 256, 8], rows=5013, grid=3, zf='rand'),
    dict(id='act1e-3', dims=[64, 256, 256, 1], rows=300, scale=1e-3),
]


@pytest.mark.parametrize('case', TC5_CASES, ids=[c['id'] for c in TC5_CASES])
def test_tc5_matches_float64(case):
    ops._stream()
    dims, rows, zf, what = case['dims'], case['rows'], case.get('zf'), 'tc5 ' + case['id']
    net = _net(dims, seed=rows, bscale=case.get('scale', 1.0))
    f = ops.Tc5Forward(net)
    f.grid = case.get('grid', 0)
    assert f.supported(rows)
    g = torch.Generator(device=DEV).manual_seed(rows)
    D = dims[0]
    x = torch.randn(rows, D, generator=g, device=DEV) * 2 + 0.5
    if zf is None:
        x[::11] = 0.0
    if zf == 'edge':
        x = _edge_x(x, g)
    x = x * case.get('scale', 1.0)
    stats = _stats(zf, D, g) if zf else None
    obuf = torch.full((rows + PADR, dims[-1] + 3), float('nan'), device=DEV)
    out = obuf[:rows, :dims[-1]]
    wn = case.get('win_n', 0)
    if wn:
        x3 = x.view(rows // (wn + 1), wn + 1, D)
        fn = lambda: f(x3[:, :wn].contiguous(), out, zf_stats=stats, x_next=x3[:, wn:].contiguous(), win_n=wn)  # noqa
    else:
        fn = lambda: f(x, out, zf_stats=stats)  # noqa: E731
    names = _forward_kernels(fn)
    _assert_family(names, 'tc5', what)
    _check_writes(obuf, rows, dims[-1], what)
    x64 = x.double()
    z, ez = _zfilter64(x64, stats, recip=True) if zf else (x64, torch.zeros_like(x64))
    worst = _check_chain(net, z, ez, None, out, C_BAR['tc5'], what)
    print('measured tc5 %s c=%.3e' % (case['id'], worst))


def test_tc5_declines_outside_its_limits():
    """MAX_K0 = 256, hidden widths multiples of 32 up to 256, 1-8 outputs, 128 rows at least."""
    for dims, rows in [([288, 256, 256, 1], 1000), ([64, 256, 256, 9], 1000), ([64, 288, 256, 1], 1000),
                       ([64, 256, 100, 1], 1000), ([48, 256, 256, 1], 1000), ([64, 256, 256, 1], 127)]:
        assert not ops.Tc5Forward(_net(dims)).supported(rows), (dims, rows)
    assert ops.Tc5Forward(_net([256, 256, 256, 8])).supported(128)


# ---- the packed cluster kernel (PackedWeights) ---------------------------------------------------------------------
PK_NETS = [('actor', dict(dims=[64, 256, 256, 8], zf='rand')),
           ('aux0-edge', dict(dims=[12, 64, 5], aux=(0, 3), zf='edge')),
           ('critic-aux1', dict(dims=[10, 200, 120, 1], aux=(1, 4))), ('wide-last', dict(dims=[33, 100, 52, 40]))]


@pytest.mark.parametrize('rows', [1, 31, 32, 33, 97])
@pytest.mark.parametrize('label,spec', PK_NETS, ids=[p[0] for p in PK_NETS])
def test_packed_matches_float64(label, spec, rows):
    ops._stream()
    dims, zf, what = spec['dims'], spec.get('zf'), 'pk %s rows %d' % (label, rows)
    net = _net(dims, aux=spec.get('aux'), seed=rows)
    pk = ops.PackedWeights(net)
    assert pk.supported
    pk.refresh()
    g = torch.Generator(device=DEV).manual_seed(rows + 5)
    D = dims[0]
    x = torch.randn(rows, D, generator=g, device=DEV) * 2 + 0.5
    if zf is None:
        x[::11] = 0.0
    if zf == 'edge':
        x = _edge_x(x, g)
    stats = _stats(zf, D, g) if zf else None
    aux64, aux = None, None
    if spec.get('aux'):
        ad = spec['aux'][1]
        abuf = torch.full((rows, ad + 3), float('nan'), device=DEV)
        abuf[:, :ad] = torch.rand(rows, ad, generator=g, device=DEV) * 2 - 1
        aux, aux64 = abuf[:, :ad], abuf[:, :ad].double()
    obuf = torch.full((rows + PADR, dims[-1] + 3), float('nan'), device=DEV)
    names = _forward_kernels(lambda: ops.mlp_forward_packed(pk, x, zf_stats=stats, zf_eps=EPS, aux=aux,
                                                            out=obuf[:rows, :dims[-1]]))
    _assert_family(names, 'pk', what)
    _check_writes(obuf, rows, dims[-1], what)
    x64 = x.double()
    z, ez = _zfilter64(x64, stats) if zf else (x64, torch.zeros_like(x64))
    worst = _check_chain(net, z, ez, aux64, obuf[:rows, :dims[-1]], C_BAR['pk'], what)
    print('measured pk %s c=%.3e' % (what, worst))


# Last in the file: once a child process has run its own CUDA activity trace, the trace of this process can miss
# kernel records, and every test above relies on that trace.
def test_tile_1_64_through_tuning_override():
    """mlp_fwd_kernel<1, 64> is reached only through SB200_FWD_TM=1 (read once per process): fits(8, 64) accepts at most
    1088 columns, and every such width already takes <2, 16> or a wider tile.  One case in a fresh process."""
    assert _widest(lambda w: _tile_fits(w, 8, 64)) < W_T2_16
    here = os.path.dirname(os.path.abspath(__file__))
    code = ('import sys; sys.path[:0] = [%r, %r]; import test_mlp_forward_envelope_gpu as t; '
            't._run_case(dict(id="tm1", family="t1_64", mode=0, rows=3000, dims=[16, 200, 40], zf="rand"))'
            % (here, os.path.dirname(here)))
    r = subprocess.run([sys.executable, '-c', code], env=dict(os.environ, SB200_FWD_TM='1'), capture_output=True,
                       text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]

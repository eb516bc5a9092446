"""Training-side kernels against float64 autograd: the backward GEMMs, MlpTrainer.backward as a chain, the loss kernels,
the optimiser step and the gradients of whole learn() calls at full size.

Parameters after Adam only show the sign of a gradient, so these tests read the gradients themselves: kernel-layout
buffers through FlatNet.get_layer(l, buf=...) / extra_view(buf), compared with tests/grad_ref.py.  Every bar quotes the
worst ratio measured on an H100 80GB HBM3 next to it."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import grad_ref as R
from helpers import ppo_configs, ddpg_configs
from surreal_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NAN = float('nan')


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _lib_():
    ops._stream()                     # sb200_init once
    return _lib.lib()


def _ints(gen, *shape, zeros=False):
    """small integers in [-3, 3]: every product and partial sum below 2^24 is exact in fp32."""
    t = torch.randint(-3, 4, shape, generator=gen, device=DEV).float()
    if zeros:
        t[torch.rand(shape, generator=gen, device=DEV) < 0.2] = 0.0
    return t


def _padded(vals, ld):
    """[rows, ld] buffer holding ``vals`` in the first columns, NaN sentinels in the padding."""
    out = torch.full((vals.shape[0], ld), NAN, device=DEV)
    out[:, :vals.shape[1]] = vals
    return out


# ------------------------------------------------------------------------------------------------------------------
# a. backward GEMMs, exact arithmetic
# (M, K, N, splits): every edge value appears; splits > ceil(M / 16) leaves slabs empty; 131072 rows with several splits
GEMM_CASES = [(1, 1, 1, 1), (15, 3, 300, 2), (16, 4, 65, 3), (17, 5, 64, 7), (63, 16, 63, 16), (64, 17, 17, 1),
              (65, 63, 16, 2), (1000, 64, 5, 3), (1000, 65, 4, 7), (17, 256, 3, 16), (65, 300, 1, 16), (1, 300, 256, 16),
              (15, 65, 300, 3), (131072, 64, 256, 16), (131072, 300, 17, 7)]


@pytest.mark.parametrize('M,K,N,splits', GEMM_CASES)
def test_linear_bwd_exact(M, K, N, splits):
    L = _lib_()
    gen = torch.Generator(device=DEV).manual_seed(M * 7 + K * 3 + N)
    ldw, ldk, ldn = ops._ru(N, 4), ops._ru(K, 4) + 4, ops._ru(N, 4) + 4
    X, dY = _ints(gen, M, K), _ints(gen, M, N)
    Xact = _ints(gen, M, K, zeros=True)                       # zeros and negatives: relu' = 0 there
    W = torch.zeros(K, ldw, device=DEV)                       # padding columns of W are zero (FlatNet invariant)
    W[:, :N] = _ints(gen, K, N)
    Xb, dYb, Xab = _padded(X, ldk), _padded(dY, ldn), _padded(Xact, ldk)
    X64, dY64, W64 = X.double(), dY.double(), W[:, :N].double()
    # dX = (dY W^T) * relu'(Xact), and without the mask (Xact = NULL)
    for use_act in (True, False):
        dX = torch.full((M, ldk), NAN, device=DEV)
        _lib.check(L.sb200_linear_bwd_dx_f32(_p(dYb), ldn, _p(W), ldw, _p(Xab if use_act else None), ldk, _p(dX), ldk,
                                             M, N, K, ops._stream()), 'dx')
        ref = dY64 @ W64.t()
        if use_act:
            ref = ref * (Xact.double() > 0)
        torch.cuda.synchronize()
        assert torch.equal(dX[:, :K].double(), ref), ('dX', use_act)
        assert bool(torch.isnan(dX[:, K:]).all()), 'dX padding columns written'
    # dW / db as `splits` slabs inside a flat buffer: the layer sits at [w, w + K*ldw) + [b, b + ldw) with guard space
    w_off = 8
    b_off = w_off + K * ldw
    size = b_off + ldw + 12
    ref_w = X64.t() @ dY64
    ref_b = dY64.sum(0)
    for with_db in (True, False):                            # db = NULL: the aux-column call
        slabs = torch.full((splits, size), NAN, device=DEV)
        _lib.check(L.sb200_linear_bwd_dw_f32(_p(Xb), ldk, _p(dYb), ldn, C.c_void_p(slabs.data_ptr() + 4 * w_off),
                                             C.c_void_p(slabs.data_ptr() + 4 * b_off) if with_db else None, size, splits,
                                             ldw, M, K, N, ops._stream()), 'dw')
        torch.cuda.synchronize()
        sw = slabs[:, w_off:b_off].view(splits, K, ldw)
        sb = slabs[:, b_off:b_off + ldw]
        assert not bool(torch.isnan(sw[:, :, :N]).any()), 'dW region left unwritten / NaN'
        assert torch.equal(sw[:, :, :N].double().sum(0), ref_w), 'dW'
        # nothing outside [w, w + K*ldw) (columns < N) and [b, b + N) is written: padding must stay as it was
        assert bool(torch.isnan(sw[:, :, N:]).all()) and bool(torch.isnan(slabs[:, :w_off]).all())
        assert bool(torch.isnan(slabs[:, b_off + N:]).all())
        if with_db:
            assert not bool(torch.isnan(sb[:, :N]).any())
            assert torch.equal(sb[:, :N].double().sum(0), ref_b), 'db'
        else:
            assert bool(torch.isnan(sb).all()), 'db written by the aux call'


# ------------------------------------------------------------------------------------------------------------------
# b. backward GEMMs, random data at the learner's shapes
@pytest.mark.parametrize('M,K,N', [(1024, 64, 256), (4096, 256, 256), (4096, 256, 8), (131072, 256, 256)])
def test_linear_bwd_random_error_bound(M, K, N):
    """|g - g64| <= c |X|^T |dY| elementwise (the standard a-priori bound of a dot product, with c in place of the
    length times the unit roundoff).  Measured worst c: dX 4.7e-7 (bar 1e-6), dW 4.7e-8 over 16 slabs (bar 2e-7)."""
    L = _lib_()
    gen = torch.Generator(device=DEV).manual_seed(M + K + N)
    splits = max(1, min(16, M // 128))
    ldw = ops._ru(N, 4)
    X = torch.randn(M, K, generator=gen, device=DEV)
    dY = torch.randn(M, N, generator=gen, device=DEV)
    W = torch.zeros(K, ldw, device=DEV)
    W[:, :N] = torch.randn(K, N, generator=gen, device=DEV) * 0.1
    slabs = torch.zeros(splits, K * ldw + ldw, device=DEV)
    _lib.check(L.sb200_linear_bwd_dw_f32(_p(X), K, _p(dY), N if N % 4 == 0 else ldw, _p(slabs),
                                         C.c_void_p(slabs.data_ptr() + 4 * K * ldw), slabs.shape[1], splits, ldw, M, K, N,
                                         ops._stream()), 'dw')
    dX = torch.zeros(M, K, device=DEV)
    _lib.check(L.sb200_linear_bwd_dx_f32(_p(dY), N, _p(W), ldw, None, 0, _p(dX), K, M, N, K, ops._stream()), 'dx')
    g = slabs.double().sum(0)
    gw = g[:K * ldw].view(K, ldw)[:, :N]
    X64, dY64 = X.double(), dY.double()
    cw = float(((gw - X64.t() @ dY64).abs() / (X64.abs().t() @ dY64.abs())).max())
    W64 = W[:, :N].double()
    cx = float(((dX.double() - dY64 @ W64.t()).abs() / (dY64.abs() @ W64.abs().t())).max())
    print('measured gemm', M, K, N, cw, cx)
    assert cw <= 2e-7 and cx <= 1e-6, (cw, cx)


# ------------------------------------------------------------------------------------------------------------------
# c. MlpTrainer.backward as a whole chain
def _rand_net(dims, acts, gen, aux_layer=-1, aux_dim=0, extra=0):
    net = ops.FlatNet(dims, acts, DEV, aux_layer=aux_layer, aux_dim=aux_dim, extra=extra)
    layers = []
    for l in range(len(dims) - 1):
        k = dims[l] + (aux_dim if aux_layer == l else 0)
        s = 1.0 / math.sqrt(k)
        layers.append(((torch.rand(dims[l + 1], k, generator=gen) * 2 - 1) * s, (torch.rand(dims[l + 1], generator=gen) * 2 - 1) * s))
    return net.load_layers(layers), layers


def _rel(got, exp):
    return float((got.double() - exp).norm()) / max(float(exp.norm()), 1e-30)


def _maxrel(got, exp):
    return float((got.double() - exp).abs().max()) / max(float(exp.abs().max()), 1e-30)


CHAIN_CASES = [([11, 32, 24, 3], -1, 0, True, 16), ([17, 300, 200, 6], -1, 0, 'linear', 77),
               ([64, 256, 256, 8], -1, 0, 'relu', 1024), ([64, 256, 256, 1], -1, 0, False, 4096),
               ([64, 400, 300, 1], 1, 8, False, 1024), ([64, 400, 300, 1], 1, 3, 'relu', 77)]


@pytest.mark.parametrize('dims,aux_layer,aux_dim,input_grad,M', CHAIN_CASES)
def test_trainer_backward_chain(dims, aux_layer, aux_dim, input_grad, M):
    """Seed d[-1] and compare the summed slabs with float64 autograd of sum(seed * pre_out), the relu masks taken
    from the trainer's own saved activations.  Measured worst per-tensor relative L2 2.0e-6, max error 2.4e-6 of
    max|g64|; bars 1e-5 / 2e-5.  SB200_OVERLAP_DW (dW GEMMs on a side stream) must not change a bit."""
    gen = torch.Generator().manual_seed(M + dims[1])
    A = dims[-1]
    acts = [ops.ACT_RELU] * (len(dims) - 2) + [ops.ACT_TANH if A > 1 else ops.ACT_NONE]
    net, layers = _rand_net(dims, acts, gen, aux_layer, aux_dim, extra=A if A > 1 else 0)
    x = torch.randn(M, dims[0], generator=gen).to(DEV)
    if input_grad:
        x = x.abs() * (torch.rand(M, dims[0], generator=gen).to(DEV) < 0.7)      # a relu output feeding the net
    aux = (torch.rand(M, aux_dim, generator=gen) * 2 - 1).to(DEV) if aux_dim else None
    seed = torch.randn(M, A, generator=gen).to(DEV)
    slabs = []
    for overlap in (False, True):
        tr = ops.MlpTrainer(net, M, 1e-3, input_grad=input_grad)
        tr.overlap_dw = overlap
        tr.forward(x, aux=aux)
        tr.d[-1].zero_()
        tr.d[-1][:, :A] = seed
        tr.backward()
        torch.cuda.synchronize()
        slabs.append(tr.slabs.clone())
    assert torch.equal(slabs[0], slabs[1]), 'SB200_OVERLAP_DW changes the slabs'
    g = slabs[0].double().sum(0).float()
    masks = [(h[:, :n] > 0) for h, n in zip(tr.h[:-1], dims[1:-1])]
    Ls = [(R.f64(w).to(DEV).requires_grad_(True), R.f64(b).to(DEV).requires_grad_(True)) for w, b in layers]
    x64 = R.f64(x).requires_grad_(True)
    a64 = R.f64(aux).requires_grad_(True) if aux is not None else None
    pre = R.trunk(x64, Ls, aux=a64, aux_layer=aux_layer, masks=masks)
    leaves = [t for wb in Ls for t in wb] + [x64] + ([a64] if a64 is not None else [])
    gs = torch.autograd.grad((pre * R.f64(seed)).sum(), leaves)
    for l in range(len(layers)):
        gw, gb = net.get_layer(l, buf=g)
        for got, exp, what in ((gw, gs[2 * l], 'W'), (gb, gs[2 * l + 1], 'b')):
            print('measured chain', dims, M, what, l, _rel(got, exp), _maxrel(got, exp))
            assert _rel(got, exp) <= 1e-5 and _maxrel(got, exp) <= 2e-5, (what, l, _rel(got, exp), _maxrel(got, exp))
    # the padding of the flat gradient stays zero (Adam runs over the whole buffer)
    for l, lay in enumerate(net.layout):
        assert float(net.W(l, buf=g)[:, lay['N']:].abs().max() if lay['ldw'] > lay['N'] else 0.0) == 0.0
        assert float(net.b(l, buf=g)[lay['N']:].abs().max() if lay['ldw'] > lay['N'] else 0.0) == 0.0
    if input_grad:
        gx = gs[2 * len(layers)]
        if input_grad != 'linear':
            gx = gx * (x > 0)
        got = tr.dx0[:, :dims[0]]
        assert _rel(got, gx) <= 1e-5 and _maxrel(got, gx) <= 2e-5, ('dx0', _rel(got, gx), _maxrel(got, gx))
    if aux is not None:
        # the DDPG actor's path: only the dX chain down to layer 1, then d loss / d aux
        tr.d[-1].zero_()
        tr.d[-1][:, :A] = seed
        tr.d[aux_layer].fill_(NAN)
        tr.backward_inputs(stop_layer=aux_layer)
        out = torch.full((M, ops._ru(aux_dim, 4)), NAN, device=DEV)
        tr.grad_wrt_aux(aux_layer, out)
        torch.cuda.synchronize()
        ga = gs[-1]
        assert _rel(out[:, :aux_dim], ga) <= 1e-5 and _maxrel(out[:, :aux_dim], ga) <= 2e-5, \
            ('aux', _rel(out[:, :aux_dim], ga), _maxrel(out[:, :aux_dim], ga))


# ------------------------------------------------------------------------------------------------------------------
# d. loss kernels
RATIOS = (0.65, 0.75, 0.9, 1.0, 1.1, 1.3, 1.6)      # 1 - eps = 0.8 and 1 + eps = 1.2 stay >= 6 % away
KAPPAS = (1.2, 2.0, 3.5, 6.0)                        # likelihood e^-0.72, e^-2, e^-6.1 (behaviour < 1e-2), e^-18 (dead)


def _policy_rows(B, A, gen):
    """Rows built per regime: |action - mean| / std = kappa along a random direction u, the behaviour mean shifted by
    s along u so that log(ratio) = s^2 / 2 - s kappa hits a chosen ratio; sum(log std) = -A log(2 pi) / 2 puts the
    likelihood at exp(-kappa^2 / 2)."""
    pre = torch.randn(B, A, generator=gen, dtype=torch.float64) * 0.7
    mean = torch.tanh(pre)
    v = torch.randn(A, generator=gen, dtype=torch.float64) * 0.2
    log_std = -0.5 * math.log(2 * math.pi) + (v - v.mean())
    std = torch.exp(log_std).expand(B, A)
    b = torch.arange(B)
    kappa = torch.tensor(KAPPAS, dtype=torch.float64)[b % 4]
    ratio = torch.tensor(RATIOS, dtype=torch.float64)[(b // 4) % 7] * (1 + 0.01 * torch.rand(B, generator=gen, dtype=torch.float64))
    sign = torch.where((b // 28) % 2 == 0, 1.0, -1.0).double()
    adv = sign * (0.2 + torch.rand(B, generator=gen, dtype=torch.float64))
    u = torch.randn(B, A, generator=gen, dtype=torch.float64)
    u = u / u.norm(dim=1, keepdim=True)
    rho = torch.log(ratio)
    s = kappa - torch.sqrt(kappa ** 2 + 2 * rho)
    actions = mean + std * kappa.view(-1, 1) * u
    behave = torch.cat([mean + std * s.view(-1, 1) * u, std], 1)
    ref = torch.cat([mean + 0.15 * std * torch.randn(B, A, generator=gen, dtype=torch.float64),
                     std * torch.exp(0.05 * torch.randn(B, A, generator=gen, dtype=torch.float64))], 1)
    return mean.float(), log_std.float(), actions.float(), adv.float(), behave.float(), ref.float()


LOSS_SHAPES = [(1, 1), (3, 255), (8, 256), (32, 257), (64, 4096), (8, 4096), (64, 1), (1, 257)]


def _stat_ok(got, exp, what, tol=1e-5):
    print('measured stat', what, tol, abs(got - exp) / max(1.0, abs(exp)))
    assert abs(got - exp) <= tol * max(1.0, abs(exp)), (what, got, exp)


@pytest.mark.parametrize('A,B', LOSS_SHAPES)
@pytest.mark.parametrize('mode', ['clip', 'adapt', 'adapt-hinge'])
def test_ppo_policy_loss_kernel(mode, A, B):
    """dpre, dlog_var and the statistics against float64 autograd.  Measured worst: dpre error 0.25 of its bar
    (1e-5 max|ref| + 1e-4 |ref|), statistics 0.4 of theirs (1e-5 max(1, |v|))."""
    L = _lib_()
    gen = torch.Generator().manual_seed(A * 1000 + B)
    mean, log_var, actions, adv, behave, ref = _policy_rows(B, A, gen)
    m_ = 0 if mode == 'clip' else 1
    D = lambda t: t.contiguous().to(DEV)  # noqa: E731
    mean_d, lv_d, act_d, adv_d, beh_d, ref_d = map(D, (mean, log_var, actions, adv, behave, ref))
    lam = 1.0
    std64 = torch.exp(R.f64(log_var)).expand(B, A)
    klm = float(R.kl(R.f64(ref[:, :A]), R.f64(ref[:, A:]), R.f64(mean), std64).mean())
    kl_target = klm / 2 * (0.7 if mode == 'adapt-hinge' else 1.4)    # 30 % away from the hinge's branch point
    hyper = torch.tensor([0.2, lam], dtype=torch.float64, device=DEV)
    ldd = ops._ru(A, 4) + 4
    ws = torch.zeros(int(L.sb200_ppo_loss_workspace_bytes(B, A)), dtype=torch.uint8, device=DEV)
    outs = []
    for call in range(2):                                # the workspace counter resets itself: a second call agrees
        dpre = torch.full((B, ldd), NAN, device=DEV)
        dlv = torch.full((A,), NAN, device=DEV)
        stats = torch.zeros(32, device=DEV)
        if m_ == 1:
            _lib.check(L.sb200_ppo_kl_f32(_p(ref_d), 2 * A, _p(mean_d), A, _p(lv_d), B, A, _p(stats), 3, 0.0, None, 0,
                                          _p(ws), ops._stream()), 'kl')
        _lib.check(L.sb200_ppo_policy_loss_f32(m_, _p(mean_d), A, _p(lv_d), _p(act_d), A, _p(adv_d), _p(beh_d), 2 * A,
                                               _p(ref_d), 2 * A, B, A, _p(hyper), 250.0, kl_target, _p(dpre), ldd,
                                               _p(dlv), _p(stats), _p(ws), None, ops._stream()), 'policy loss')
        torch.cuda.synchronize()
        outs.append((dpre.clone(), dlv.clone(), stats.clone()))
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b), 'second call differs'
    dpre, dlv, stats = outs[0]
    hp = dict(clip_eps=0.2) if m_ == 0 else dict(ref=ref, beta=lam, kl_target=kl_target, eta=250.0)
    r = R.policy_loss_head(torch.atanh(R.f64(mean)), log_var, actions, adv, behave, 'clip' if m_ == 0 else 'adapt', **hp)
    if m_ == 1:
        assert r['hinge'] == (mode == 'adapt-hinge')
    gp = r['g_pre'].to(DEV)
    err = (dpre[:, :A].double() - gp).abs()
    print('measured dpre', mode, A, B, float((err / (1e-5 * float(gp.abs().max()) + 1e-4 * gp.abs())).max()))
    assert bool((err <= 1e-5 * float(gp.abs().max()) + 1e-4 * gp.abs()).all()), float(err.max())
    assert bool((dpre[:, A:] == 0).all()), 'dpre padding must come back as zero'
    gl = r['g_log_var'].to(DEV)
    el = (dlv.double() - gl).abs()
    assert bool((el <= 1e-5 * float(gl.abs().max()) + 1e-4 * gl.abs()).all()), float(el.max())
    s = stats.cpu().tolist()
    _stat_ok(s[0], float(r['surr']), 'surr')
    if m_ == 0:
        _stat_ok(s[1], float(r['loss']), 'loss')
    else:
        # the KL sums 2A terms of order 1 and subtracts A / 2 in fp32 (as the oracle does): its absolute rounding,
        # ~A ulp, reaches the loss times d loss / d KL = beta + 2 eta (KL - 2 kl_target)^+.  Measured worst 0.24 of tol.
        slope = lam + 2 * 250.0 * max(0.0, float(r['kl']) - 2 * kl_target)
        tol = 1e-5 * max(1.0, abs(float(r['loss']))) + slope * A * 2.4e-7
        print('measured adaptloss', abs(s[1] - float(r['loss'])) / tol)
        assert abs(s[1] - float(r['loss'])) <= tol, ('loss', s[1], float(r['loss']), tol)
    _stat_ok(s[2], float(r['entropy']), 'entropy')
    if m_ == 1:
        _stat_ok(s[3], float(r['kl']), 'kl')
    # a raised stop flag writes nothing
    stop = torch.ones(1, dtype=torch.int32, device=DEV)
    dpre2, dlv2, st2 = torch.full_like(dpre, 7.0), torch.full_like(dlv, 7.0), torch.full_like(stats, 7.0)
    _lib.check(L.sb200_ppo_kl_f32(_p(ref_d), 2 * A, _p(mean_d), A, _p(lv_d), B, A, _p(st2), 3, 0.0, _p(stop), 0, _p(ws),
                                  ops._stream()), 'kl')
    _lib.check(L.sb200_ppo_policy_loss_f32(m_, _p(mean_d), A, _p(lv_d), _p(act_d), A, _p(adv_d), _p(beh_d), 2 * A,
                                           _p(ref_d), 2 * A, B, A, _p(hyper), 250.0, kl_target, _p(dpre2), ldd, _p(dlv2),
                                           _p(st2), _p(ws), _p(stop), ops._stream()), 'policy loss')
    torch.cuda.synchronize()
    assert bool((dpre2 == 7.0).all() and (dlv2 == 7.0).all() and (st2 == 7.0).all())


GRAD_BAR, STAT_BAR = 4e-7, 4e-7


def _grad_ok(got, exp, what):
    e = float((got.cpu().double() - exp).abs().max()) / max(float(exp.abs().max()), 1e-30)
    print('measured lossgrad', what, e)
    assert e <= GRAD_BAR, (what, e)


@pytest.mark.parametrize('B', [1, 255, 256, 257, 4096])
def test_value_and_ddpg_loss_kernels(B):
    """sb200_value_loss_f32, sb200_ddpg_critic_loss_f32, sb200_ddpg_actor_seed_f32 and sb200_tanh_bwd_f32 against the
    float64 helpers.  Gradients: elementwise error / max|ref|, measured worst 6.8e-8 (bar 4e-7).  Statistics:
    error / max(1, |v|), measured worst 4.9e-8 (bar 4e-7)."""
    L = _lib_()
    gen = torch.Generator().manual_seed(B)
    ldd = 8
    v = torch.randn(B, 1, generator=gen)
    ret = torch.randn(B, generator=gen) * 2 + 0.5
    v_d, ret_d = v.to(DEV), ret.to(DEV)
    ws = torch.zeros(int(L.sb200_ppo_loss_workspace_bytes(B, 1)), dtype=torch.uint8, device=DEV)
    dpre = torch.full((B, ldd), NAN, device=DEV)
    stats = torch.zeros(32, device=DEV)
    _lib.check(L.sb200_value_loss_f32(_p(v_d), 1, _p(ret_d), B, _p(dpre), ldd, _p(stats), _p(ws),
                                      ops._stream()), 'value loss')
    torch.cuda.synchronize()
    v64 = R.f64(v).requires_grad_(True)
    loss = (v64 - R.f64(ret).view(-1, 1)).pow(2).mean()
    g, = torch.autograd.grad(loss, v64)
    _grad_ok(dpre[:, :1], g, 'value')
    assert bool((dpre[:, 1:] == 0).all())
    s = stats.cpu().tolist()
    _stat_ok(s[6], float(loss), 'val loss', tol=STAT_BAR)
    _stat_ok(s[9], float(ret.double().mean()), 'return mean', tol=STAT_BAR)
    if B > 1:
        ev = 1 - torch.var(R.f64(ret) - R.f64(v).view(-1)) / torch.var(R.f64(ret))
        _stat_ok(s[7], float(ev), 'explained var', tol=STAT_BAR)
    # DDPG critic MSE and actor seed
    dws = torch.zeros(int(L.sb200_ddpg_workspace_bytes(B)), dtype=torch.uint8, device=DEV)
    q, y = torch.randn(B, 1, generator=gen), torch.randn(B, generator=gen)
    q_d, y_d = q.to(DEV), y.to(DEV)
    dq = torch.full((B, ldd), NAN, device=DEV)
    dst = torch.zeros(16, device=DEV)
    _lib.check(L.sb200_ddpg_critic_loss_f32(_p(q_d), 1, _p(y_d), B, _p(dq), ldd, _p(dst), _p(dws),
                                            ops._stream()), 'critic loss')
    torch.cuda.synchronize()
    r = R.ddpg_critic([(torch.eye(1), torch.zeros(1))], q, torch.zeros(B, 0), y, aux_layer=0)
    gq = r['g_pre']
    _grad_ok(dq[:, :1], gq, 'critic')
    assert bool((dq[:, 1:] == 0).all())
    _stat_ok(float(dst[1]), float(r['loss']), 'critic loss', tol=STAT_BAR)
    _stat_ok(float(dst[5]), float(r['q_mean']), 'Q_policy', tol=STAT_BAR)
    dq.fill_(NAN)
    _lib.check(L.sb200_ddpg_actor_seed_f32(_p(q_d), 1, B, _p(dq), ldd, _p(dst), _p(dws), ops._stream()), 'seed')
    torch.cuda.synchronize()
    assert bool((dq[:, 0].cpu().double() == torch.tensor(-1.0 / B, dtype=torch.float32).double()).all())
    assert bool((dq[:, 1:] == 0).all())
    _stat_ok(float(dst[0]), -float(q.double().mean()), 'actor loss', tol=STAT_BAR)
    # tanh backward with every stride different from A
    for A in (1, 3, 8):
        out = torch.tanh(torch.randn(B, A, generator=gen) * 1.5)
        dout = torch.randn(B, A, generator=gen)
        outb, doutb = _padded(out.to(DEV), A + 5), _padded(dout.to(DEV), A + 2)
        dp = torch.full((B, ops._ru(A, 4) + 4), NAN, device=DEV)
        _lib.check(L.sb200_tanh_bwd_f32(_p(doutb), A + 2, _p(outb), A + 5, B, A, _p(dp), dp.shape[1], ops._stream()), 'tanh')
        torch.cuda.synchronize()
        exp = R.f64(dout) * (1 - R.f64(out) ** 2)
        _grad_ok(dp[:, :A], exp, 'tanh')
        assert bool((dp[:, A:] == 0).all())


# ------------------------------------------------------------------------------------------------------------------
# e. optimiser
def _ulp(t):
    return torch.from_numpy(np.spacing(np.abs(t.numpy()).astype(np.float32))).float()


@pytest.mark.parametrize('n,splits,clip_mode,wd', [(4, 1, 1, 0.0), (1024, 5, 2, 1e-3), (1028, 16, 0, 1e-3),
                                                   (264 * 1024 + 4, 5, 1, 1e-3), (264 * 1024 + 4, 16, 2, 0.0),
                                                   (1028, 1, 1, 0.0)])
def test_reduce_and_adam_vs_torch(n, splits, clip_mode, wd):
    """25 steps of grad_reduce_norm + clip_adam against torch.optim.Adam(foreach=False) in fp32, preceded by
    clip_grad_norm_(5.0) / clip_grad_value_(0.01) / nothing.  Torch's addcdiv_ divides before it scales and the kernel
    scales before it divides, so results differ by rounding.  Parameters: measured worst 3.5 (ulp(p) + ulp(lr)) per
    step, with norm clipping and weight decay (1.0 elsewhere); bar 16.  Moments: measured 2.5e-6 relative L2 in that
    case (the clip coefficient, from torch's fp32 norm and the kernel's fp64 one, differs by rounding, and weight decay
    cancelling part of the clipped gradient amplifies it; 1.2e-7 elsewhere); bar 1e-5.  norm_out against the float64
    norm: measured 5.2e-8 relative; bar 3e-7."""
    L = _lib_()
    gen = torch.Generator().manual_seed(n + splits)
    steps, lr = 25, 1e-3
    p0 = torch.randn(n, generator=gen)
    p_dev, m_dev, v_dev = p0.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    grad_dev = torch.zeros(n, device=DEV)
    ws = torch.zeros(int(L.sb200_optim_workspace_bytes()), dtype=torch.uint8, device=DEV)
    lr_dev = torch.tensor([lr], dtype=torch.float64, device=DEV)
    norm_out = torch.zeros(1, device=DEV)
    pt = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([pt], lr=lr, weight_decay=wd, foreach=False)
    base = torch.randn(n, generator=gen)
    base[::7] = 0.0                                        # exact zeros: eps dominates the step
    tiny = 1e-9 * torch.sign(torch.randn(n, generator=gen)[3::11])
    scales = [0.02, 0.3, 0.05, 1.0, 0.01] * 5              # the global norm is above 5 on some steps, below on others
    worst_p = worst_m = worst_n = 0.0
    for t in range(steps):
        slabs = (base * scales[t] * math.sqrt(4096.0 / n)).repeat(splits, 1) / splits
        slabs += torch.randn(splits, n, generator=gen) * 1e-3 * scales[t]
        slabs[:, ::7] = 0.0
        slabs[:, 3::11] = tiny / splits                    # ~1e-9 gradients: eps dominates the step there too
        slabs_d = slabs.to(DEV)
        _lib.check(L.sb200_grad_reduce_norm_f32(_p(slabs_d), n, splits, _p(grad_dev), n, 1.0, 1, _p(ws), None,
                                                ops._stream()), 'reduce')
        _lib.check(L.sb200_clip_adam_f32(_p(p_dev), _p(grad_dev), _p(m_dev), _p(v_dev), n, _p(lr_dev), 0.9, 0.999, 1e-8,
                                         wd, clip_mode, 5.0 if clip_mode == 1 else 0.01, _p(ws), _p(norm_out), None,
                                         ops._stream()), 'adam')
        g = slabs[0].clone()
        for z in range(1, splits):
            g += slabs[z]                                  # the kernel's fixed summation order: bit-identical
        torch.cuda.synchronize()
        assert torch.equal(grad_dev.cpu(), g), 'reduced gradient'
        n64 = float(slabs.double().sum(0).norm())
        worst_n = max(worst_n, abs(float(norm_out) - n64) / n64)
        assert abs(float(norm_out) - n64) <= 3e-7 * n64, (float(norm_out), n64)
        pt.grad = g.clone()
        if clip_mode == 1:
            torch.nn.utils.clip_grad_norm_([pt], 5.0)
        elif clip_mode == 2:
            torch.nn.utils.clip_grad_value_([pt], 0.01)
        opt.step()
        # per step: one rounding of p + update (an ulp of p) and a few ulp of the update itself (<= lr)
        dp = (p_dev.cpu() - pt.detach()).abs() / ((t + 1) * (_ulp(pt.detach()) + float(np.spacing(np.float32(lr)))))
        worst_p = max(worst_p, float(dp.max()))
        assert float(dp.max()) <= 16, ('params', t, float(dp.max()))
        st = opt.state[pt]
        for got, exp in ((m_dev, st['exp_avg']), (v_dev, st['exp_avg_sq'])):
            e = float((got.cpu().double() - exp.double()).norm()) / max(float(exp.double().norm()), 1e-30)
            worst_m = max(worst_m, e)
            assert e <= 1e-5, ('moments', t, e)
    # which steps clipped: the global norm crosses 5.0
    print('measured adam', n, splits, clip_mode, wd, 'params', worst_p, 'moments', worst_m, 'norm', worst_n)
    if clip_mode == 1:
        norms = [float((base * s * math.sqrt(4096.0 / n)).norm()) for s in scales[:5]]
        assert min(norms) < 5.0 < max(norms)


def test_optimizer_stop_flag_and_state_dict_continuation():
    """A raised stop flag turns reduce and Adam into no-ops (the device step counter does not move); a run split by
    state_dict() / load_state_dict() equals an unbroken run bit for bit (the bias correction continues)."""
    gen = torch.Generator().manual_seed(9)
    net, _ = _rand_net([13, 40, 5], [ops.ACT_RELU, ops.ACT_TANH], gen, extra=5)
    grads = [torch.randn(3, net.size, generator=gen).to(DEV) * 0.1 for _ in range(12)]

    def run(tr, gs):
        for g in gs:
            tr.slabs.copy_(g)
            tr.step()

    a = ops.MlpTrainer(net.clone_like(), 16, 1e-3, clip_mode=1, clip_value=5.0, splits=3)
    run(a, grads)
    b = ops.MlpTrainer(net.clone_like(), 16, 1e-3, clip_mode=1, clip_value=5.0, splits=3)
    run(b, grads[:5])
    sd = b.state_dict()
    c = ops.MlpTrainer(ops.FlatNet(net.dims, net.acts, DEV, extra=5), 16, 1e-3, clip_mode=1, clip_value=5.0, splits=3)
    c.net.params.copy_(b.net.params)
    c.load_state_dict(sd)
    before = (c.net.params.clone(), c.exp_avg.clone(), c.exp_avg_sq.clone(), c.ws.clone(), c.grad.clone())
    stop = torch.ones(1, dtype=torch.int32, device=DEV)
    c.slabs.copy_(grads[5])
    c.step(stop_flag=stop)
    torch.cuda.synchronize()
    for x, y in zip(before, (c.net.params, c.exp_avg, c.exp_avg_sq, c.ws, c.grad)):
        assert torch.equal(x, y), 'stop flag: a kernel wrote'
    run(c, grads[5:])
    torch.cuda.synchronize()
    assert torch.equal(a.net.params, c.net.params) and torch.equal(a.exp_avg, c.exp_avg) and \
        torch.equal(a.exp_avg_sq, c.exp_avg_sq)


# ------------------------------------------------------------------------------------------------------------------
# f. full-size gradients of one learn()
def _layers(dims, gen, aux=0, aux_layer=-1):
    out = []
    for i in range(len(dims) - 1):
        k = dims[i] + (aux if aux_layer == i else 0)
        b = 1.0 / np.sqrt(k)
        out.append(((torch.rand(dims[i + 1], k, generator=gen) * 2 - 1) * b, (torch.rand(dims[i + 1], generator=gen) * 2 - 1) * b))
    return out


LEARN_BAR = 1e-4


def _check_grads(net, buf, ref_grads, what, extra=None, bar=LEARN_BAR):
    """per tensor: relative L2 <= bar and max error <= bar max|g64|.  LEARN_BAR (whole learn() calls): measured worst
    4.4e-5 / 4.4e-5, the DDPG critic's output bias, a sum of 4096 terms of both signs; PPO actor 3.4e-5 / 3.8e-5
    (adapt, one-launch learner)."""
    g = buf.detach()
    worst = []
    for l, (rw, rb) in enumerate(ref_grads):
        gw, gb = net.get_layer(l, buf=g)
        for got, exp, nm in ((gw, rw, 'W'), (gb, rb, 'b')):
            exp = exp.to(got.device)
            worst.append((_rel(got, exp), _maxrel(got, exp)))
            assert worst[-1][0] <= bar and worst[-1][1] <= bar, (what, nm, l, worst[-1])
    if extra is not None:
        got, exp = net.extra_view(g), extra.to(g.device)
        worst.append((_rel(got, exp), _maxrel(got, exp)))
        assert worst[-1][0] <= bar and worst[-1][1] <= bar, (what, 'log_var', worst[-1])
    print('measured', what, max(w[0] for w in worst), max(w[1] for w in worst))
    return worst


def _dev(layers):
    return [(w.to(DEV), b.to(DEV)) for w, b in layers]


def _clear_relu_ties(obs0, nets, tol=2e-5, gen=None):
    """Redraw the rows whose float64 pre-activations come within ``tol`` of 0 somewhere (a relu there could go either
    way in fp32).  nets: [(layers, transform)]."""
    for _ in range(50):
        bad = torch.zeros(obs0.shape[0], dtype=torch.bool)
        for layers, tf in nets:
            bad |= (R.hidden_margin(tf(obs0), layers) < tol).cpu()
        if not bool(bad.any()):
            return obs0
        obs0[bad] = torch.randn(int(bad.sum()), obs0.shape[1], generator=gen) * 1.2
    raise AssertionError('could not clear relu ties')


@pytest.mark.parametrize('B,n', [(1024, 128), (4096, 64)])
@pytest.mark.parametrize('mode', ['clip', 'adapt', 'adapt-hinge'])
@pytest.mark.parametrize('path', ['0', '2'])
def test_ppo_learn_gradients_fullsize(path, mode, B, n, monkeypatch):
    """One policy and one value step (epoch_policy = epoch_baseline = 1) of configs[1] and a 4096-window batch on the
    launch chain (SB200_EPOCH_KERNEL=0) and the one-launch learner (=2): actor_optim.grad / critic_optim.grad hold the
    pre-clip gradient of that step, compared with float64 autograd on the learner's own advantages / returns, the
    z-filter statistics before learn() and the reference policy."""
    from surreal_b200.learner import PPOLearner
    monkeypatch.setenv('SB200_EPOCH_KERNEL', path)
    D, A = 64, 8
    gen = torch.Generator().manual_seed(B + n + len(mode))
    al, cl = _layers([D, 256, 256, A], gen), _layers([D, 256, 256, 1], gen)
    log_var = torch.zeros(1, A) - 1.0
    zs = torch.cat([torch.randn(D, generator=gen) * 50, 500 * (1.5 + torch.rand(D, generator=gen)), torch.tensor([500.0])])
    zf = lambda x: R.zfilter(x, zs)  # noqa: E731
    rng = np.random.default_rng(B + n)
    obs = (rng.standard_normal((B, n, D)) * 1.2).astype(np.float32)
    obs[:, 0] = _clear_relu_ties(torch.from_numpy(obs[:, 0].copy()), [(al, zf), (cl, zf)], gen=gen).numpy()
    obs_next = (rng.standard_normal((B, 1, D)) * 1.2).astype(np.float32)
    with torch.no_grad():
        pd0 = torch.cat([torch.tanh(R.trunk(zf(torch.from_numpy(obs[:, 0])), [(R.f64(w), R.f64(b)) for w, b in al])),
                         torch.exp(R.f64(log_var)).expand(B, A)], 1).float().numpy()
    pd = np.tile(pd0[:, None, :], (1, n, 1)).astype(np.float32)
    pd[:, :, A:] *= np.exp(rng.uniform(-0.25, 0.25, (B, 1, 1))).astype(np.float32)
    actions = np.clip(rng.standard_normal((B, n, A)) * pd[:, :, A:] + pd[:, :, :A], -1, 1).astype(np.float32)
    rewards = rng.standard_normal((B, n)) * 0.3
    dones = np.zeros((B, n), dtype=np.float32)
    dones[rng.random(B) < 0.3, n - 1] = 1
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=(256, 256), critic_h=(256, 256), n_step=n, stride=n, B=B,
                             mode='clip' if mode == 'clip' else 'adapt')
    lc.algo.consts.epoch_policy = 1
    lc.algo.consts.epoch_baseline = 1
    L = PPOLearner(lc, ec, sc)
    assert L.epoch_policy == 1 and L.epoch_baseline == 1 and L.use_epoch_kernel == (path != '0')
    L.model.actor.load_layers(al, extra=log_var)
    L.model.critic.load_layers(cl)
    L.model.z_stats.copy_(zs.to(DEV))
    L.ref_target_model.update_target_params(L.model)
    ref_layers = al
    if mode != 'clip':
        # a reference policy away from the learner's, so that beta KL has a gradient of its own; with 'adapt-hinge' far
        # enough that the pre-step KL is above 2 kl_target (the hinge term is active), with 'adapt' below it
        shift = 0.08 if mode == 'adapt-hinge' else 0.02
        ref_layers = [(w, b) for w, b in al[:2]] + [(al[2][0], al[2][1] + shift * torch.sign(torch.randn(A, generator=gen)))]
        L.ref_target_model.actor.load_layers(ref_layers, extra=log_var)
    z_before = L.model.z_stats.clone()
    st = L.learn({'obs': obs, 'obs_next': obs_next, 'actions': actions, 'rewards': rewards, 'dones': dones,
                  'persistent_infos': [pd], 'onetime_infos': None})
    torch.cuda.synchronize()
    if path != '0':
        assert L._ek is not None and L._ek[3] is not None, 'the one-launch learner did not take this shape'
    x = R.zfilter(torch.from_numpy(obs[:, 0]).to(DEV), z_before)
    adv, ret = L._adv.view(-1), L._ret.view(-1)
    behave = torch.from_numpy(pd[:, 0]).to(DEV)
    act0 = torch.from_numpy(actions[:, 0]).to(DEV)
    with torch.no_grad():
        ref_pd = torch.cat([torch.tanh(R.trunk(x, [(R.f64(w).to(DEV), R.f64(b).to(DEV)) for w, b in ref_layers])),
                            torch.exp(R.f64(log_var)).to(DEV).expand(B, A)], 1)
    al_d, cl_d, lv_d = _dev(al), _dev(cl), log_var.to(DEV)
    if mode == 'clip':
        r = R.ppo_policy(al_d, lv_d, x, act0, adv, behave, 'clip', clip_eps=L.clip_epsilon)
    else:
        r = R.ppo_policy(al_d, lv_d, x, act0, adv, behave, 'adapt', ref=ref_pd, beta=L.beta, kl_target=L.kl_target,
                         eta=L.eta)
        assert r['hinge'] == (mode == 'adapt-hinge')
        assert abs(float(r['kl']) - 2 * L.kl_target) > 1e-3 * 2 * L.kl_target and float(r['kl']) > 1e-3
    _check_grads(L.model.actor, L.actor_optim.grad, r['grads'], 'actor', extra=r['g_log_var'])
    rv = R.value(cl_d, x, ret)
    _check_grads(L.model.critic, L.critic_optim.grad, rv['grads'], 'critic')
    na = math.sqrt(sum(float(g.pow(2).sum()) for wb in r['grads'] for g in wb) + float(r['g_log_var'].pow(2).sum()))
    nc = math.sqrt(sum(float(g.pow(2).sum()) for wb in rv['grads'] for g in wb))
    # gradient norms: measured worst 3.8e-6 relative (bar GN_BAR = 1e-5)
    print('measured gradnorm', abs(st['grad_norm_actor'] - na) / na, abs(st['grad_norm_critic'] - nc) / nc)
    assert abs(st['grad_norm_actor'] - na) <= GN_BAR * na, (st['grad_norm_actor'], na)
    assert abs(st['grad_norm_critic'] - nc) <= GN_BAR * nc, (st['grad_norm_critic'], nc)


GN_BAR = 1e-5


def test_ddpg_learn_gradients_fullsize():
    """configs[2] (B 4096, D 64, A 8, actor 300-200, critic 400-300 with the action at layer 1): the critic gradient
    of one learn() and the actor gradient through the UPDATED critic's aux columns, grad_wrt_aux and tanh_bwd, against
    float64 autograd.  The one-step parameter comparison of test_fullsize_gpu.py sees only gradient signs."""
    from surreal_b200.learner import DDPGLearner
    D, A, B = 64, 8, 4096
    lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=(300, 200), critic_h=(400, 300), B=B, n_step=3, memory_size=8192,
                              start=B)
    L = DDPGLearner(lc, ec, sc)
    gen = torch.Generator().manual_seed(11)
    al = _layers([D, 300, 200, A], gen)
    cl = _layers([D, 400], gen) + _layers([400 + A, 300, 1], gen)
    for m in (L.model, L.model_target):
        m.actor.load_layers(al)
        m.critic.load_layers(cl)
    obs = torch.randn(B, D, generator=gen)
    act = torch.rand(B, A, generator=gen) * 2 - 1
    for _ in range(50):                                 # redraw rows with a float64 pre-activation within 2e-5 of 0
        bad = (R.hidden_margin(obs, al) < 2e-5) | (R.hidden_margin(obs, cl, aux=act, aux_layer=1) < 2e-5)
        if not bool(bad.any()):
            break
        obs[bad] = torch.randn(int(bad.sum()), D, generator=gen)
        act[bad] = torch.rand(int(bad.sum()), A, generator=gen) * 2 - 1
    assert not bool(bad.any())
    obs_next = torch.randn(B, D, generator=gen)
    rew, done = torch.randn(B, 1, generator=gen), (torch.rand(B, 1, generator=gen) < 0.05).float()
    L.learn({'obs': obs.numpy(), 'obs_next': obs_next.numpy(), 'actions': act.numpy(), 'rewards': rew.numpy(),
             'dones': done.numpy()})
    torch.cuda.synchronize()
    # the Bellman target is the learner's own (its parity is tested elsewhere)
    rc = R.ddpg_critic(_dev(cl), obs.to(DEV), act.to(DEV), L._y)
    _check_grads(L.model.critic, L.critic_optim.grad, rc['grads'], 'critic')
    # the actor step ran through the updated critic: its last forward (q_pi) left its activations in the trainers
    ct, at = L.critic_optim, L.actor_optim
    crit_new = [tuple(t.cpu() for t in L.model.critic.get_layer(l)) for l in range(3)]
    cm = [(ct.h[0][:, :400] > 0), (ct.h[1][:, :300] > 0)]
    am = [(at.h[0][:, :300] > 0), (at.h[1][:, :200] > 0)]
    ra = R.ddpg_actor([(w.to(DEV), b.to(DEV)) for w, b in al], [(w.to(DEV), b.to(DEV)) for w, b in crit_new], obs.to(DEV),
                      actor_masks=am, critic_masks=cm)
    _check_grads(L.model.actor, L.actor_optim.grad, ra['grads'], 'actor')


# (actor dims, critic dims, rows, mode, grids).  The grid sets epoch2's row splits s = min(G // blocks, splits, M // 64),
# blocks = sum over both nets of ceil(H1 / 16) + ceil(D / 16) + 1: the 1000-row case runs s = 1, 2, 3, 4 over 63 row
# blocks (2 and 4 do not divide it), the 200-row case s = 3 and 1, the 515-row case (A = 32, E2_MAX_OUT) s = 1 and 8; the
# 3-row case is one row block with a one-unit head and widths 1 and 3 mod 4.
E2_CASES = [([17, 300, 200, 6], [17, 100, 68, 1], 200, 'clip', (132, 40)),
            ([17, 300, 200, 6], [17, 100, 68, 1], 1000, 'adapt-hinge', (16, 64, 100, 132)),
            ([20, 64, 64, 1], [20, 64, 64, 1], 77, 'adapt', (7, 132)),
            ([24, 64, 48, 32], [24, 64, 48, 1], 515, 'clip', (24, 132)),
            ([5, 17, 15, 1], [5, 15, 17, 1], 3, 'adapt', (1, 132))]
E2_BAR = 3e-5


@pytest.mark.parametrize('case', range(len(E2_CASES)))
def test_epoch_pair_gradients_ragged(case):
    """The one-launch learner (EpochPair built on device buffers) at ragged shapes and several grid sizes: one policy and
    one value step, actor / critic gradients and both gradient norms against float64 autograd.  Per tensor, measured
    worst relative L2 / max error 4.0e-6 / 5.5e-6 (bar E2_BAR = 3e-5); gradient norms 2.9e-6 (bar GN_BAR = 1e-5)."""
    ad, cd, M, mode, grids = E2_CASES[case]
    A, D = ad[-1], ad[0]
    gen = torch.Generator().manual_seed(100 + case)
    al, cl = _layers(ad, gen), _layers(cd, gen)
    log_var = torch.full((1, A), -1.0) + 0.2 * torch.rand(1, A, generator=gen)
    x = _clear_relu_ties(torch.randn(M, D, generator=gen) * 1.2, [(al, R.f64), (cl, R.f64)], gen=gen)
    with torch.no_grad():
        mean = torch.tanh(R.trunk(R.f64(x), [(R.f64(w), R.f64(b)) for w, b in al]))
    std = torch.exp(R.f64(log_var)).expand(M, A)
    g64 = lambda *sh: torch.randn(*sh, generator=gen, dtype=torch.float64)  # noqa: E731
    bm = (mean + 0.3 * std * g64(M, A)).clamp(-0.99, 0.99)
    bs = std * torch.exp(0.2 * g64(M, 1))
    actions = (bm + 0.5 * bs * g64(M, A)).float()
    behave = torch.cat([bm, bs], 1).float()
    ref = torch.cat([mean + 0.2 * std * g64(M, A), std], 1).float()
    adv, ret = torch.randn(M, generator=gen), torch.randn(M, generator=gen)
    m_ = 0 if mode == 'clip' else 1
    klm = float(R.kl(R.f64(ref[:, :A]), R.f64(ref[:, A:]), mean, std).mean())
    kl_target = klm / 2 * (0.7 if mode == 'adapt-hinge' else 1.4)        # 30 % away from the hinge's branch point
    hp = dict(clip_eps=0.2) if m_ == 0 else dict(ref=ref, beta=1.0, kl_target=kl_target, eta=250.0)
    r = R.ppo_policy(al, log_var, x, actions, adv, behave, 'clip' if m_ == 0 else 'adapt', **hp)
    if m_ == 1:
        assert r['hinge'] == (mode == 'adapt-hinge')
    rv = R.value(cl, x, ret)
    na = math.sqrt(sum(float(g.pow(2).sum()) for wb in r['grads'] for g in wb) + float(r['g_log_var'].pow(2).sum()))
    nc = math.sqrt(sum(float(g.pow(2).sum()) for wb in rv['grads'] for g in wb))
    dv = lambda t: t.contiguous().to(DEV)  # noqa: E731
    x_d, act_d, adv_d, beh_d, ref_d, ret_d = map(dv, (x, actions, adv, behave, ref, ret))
    hyper = torch.tensor([0.2, 1.0], dtype=torch.float64, device=DEV)
    for grid in grids:
        an = ops.FlatNet(ad, [ops.ACT_RELU, ops.ACT_RELU, ops.ACT_TANH], DEV, extra=A).load_layers(al, extra=log_var)
        cn = ops.FlatNet(cd, [ops.ACT_RELU, ops.ACT_RELU, ops.ACT_NONE], DEV).load_layers(cl)
        at = ops.MlpTrainer(an, M, 1e-3, clip_mode=1, clip_value=5.0, splits=16)
        ct = ops.MlpTrainer(cn, M, 1e-3, clip_mode=1, clip_value=5.0, splits=16)
        stats, norms = torch.zeros(32, device=DEV), torch.zeros(2, device=DEV)
        pk = ops.EpochKernel(at, m_, x_d, D, M, None, 1e-5, stats, 1, norm_out=norms[0:1], actions=act_d, lda=A, adv=adv_d,
                             behave_pd=beh_d, ldb=2 * A, ref_pd=ref_d, ldr=2 * A, hyper=hyper, eta=250.0,
                             kl_target=kl_target, grid=grid)
        vk = ops.EpochKernel(ct, 2, x_d, D, M, None, 1e-5, stats, 1, norm_out=norms[1:2], returns=ret_d)
        assert ops.EpochPair.supported(pk, vk), 'the one-launch learner rejects this shape'
        ops.EpochPair(pk, vk).run()
        torch.cuda.synchronize()
        _check_grads(an, at.grad, r['grads'], 'e2 actor grid %d' % grid, extra=r['g_log_var'], bar=E2_BAR)
        _check_grads(cn, ct.grad, rv['grads'], 'e2 critic grid %d' % grid, bar=E2_BAR)
        ga, gc = float(norms[0]), float(norms[1])
        print('measured e2norm', abs(ga - na) / na, abs(gc - nc) / nc)
        assert abs(ga - na) <= GN_BAR * na and abs(gc - nc) <= GN_BAR * nc, (ga, na, gc, nc)

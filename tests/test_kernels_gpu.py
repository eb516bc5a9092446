"""GPU parity tests: CUDA kernels (through the C-ABI) vs the CPU oracle and the golden fixtures."""
import numpy as np
import pytest
import torch

from oracle import nets as onets
from oracle.filters import ZFilter as OZFilter
from oracle.gae import gae_from_values

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device('cuda:0')


def rms(x):
    return float(x.double().pow(2).mean().sqrt())


def assert_close_scale(got, exp, tol=1e-5, what=''):
    """max|a-b| <= tol * max(1, rms(b))   (BASELINE.md §5)."""
    got, exp = got.detach().cpu().double(), exp.detach().cpu().double()
    err = float((got - exp).abs().max())
    lim = tol * max(1.0, rms(exp))
    assert err <= lim, '%s: max err %.3e > %.3e' % (what, err, lim)


def _rand_layers(dims, gen, aux_layer=-1, aux_dim=0):
    layers = []
    for l in range(len(dims) - 1):
        k = dims[l] + (aux_dim if aux_layer == l else 0)
        bound = 1.0 / np.sqrt(k)
        w = (torch.rand(dims[l + 1], k, generator=gen) * 2 - 1) * bound
        b = (torch.rand(dims[l + 1], generator=gen) * 2 - 1) * bound
        layers.append((w, b))
    return layers


@pytest.mark.parametrize('dims,rows,zf', [
    ([11, 32, 24, 3], 37, True),          # all-narrow layers, ragged rows
    ([64, 256, 256, 8], 1024, True),      # cfg2 actor
    ([64, 256, 256, 1], 3000, False),     # cfg2 critic, rows not a tile multiple
    ([17, 300, 200, 6], 333, True),       # reference default hidden sizes (K, N not multiples of 16/256)
    ([9, 40, 1], 5, False),               # 2-layer net
    ([64, 256, 256, 1], 20000, True),     # large-M tile path (BM=64)
])
def test_mlp_forward_matches_oracle(dims, rows, zf):
    from surreal_b200 import ops
    gen = torch.Generator().manual_seed(sum(dims) + rows)
    layers = _rand_layers(dims, gen)
    acts = [ops.ACT_RELU] * (len(dims) - 2) + [ops.ACT_TANH if dims[-1] > 1 else ops.ACT_NONE]
    x = torch.randn(rows, dims[0], generator=gen) * 2 + 0.5
    ozf = None
    stats = None
    if zf:
        ozf = OZFilter(dims[0])
        ozf.update(torch.randn(200, dims[0], generator=gen) * 1.7 + 0.4)
        stats = torch.cat([ozf.running_sum, ozf.running_sumsq, ozf.count]).to(_dev())
    net = ops.FlatNet(dims, acts, _dev()).load_layers(layers)
    outs = ops.mlp_forward(net, x.to(_dev()), zf_stats=stats, save_all=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        h = ozf.forward(x) if zf else x
        exp = []
        for l, (w, b) in enumerate(layers):
            h = torch.nn.functional.linear(h, w, b)
            h = torch.relu(h) if acts[l] == ops.ACT_RELU else (torch.tanh(h) if acts[l] == ops.ACT_TANH else h)
            exp.append(h)
    assert len(outs) == len(exp)
    for l, (o, e) in enumerate(zip(outs, exp)):
        assert o.shape == e.shape
        assert_close_scale(o, e, 1e-5, 'layer %d' % l)


@pytest.mark.parametrize('dims,rows,zf,aux', [
    ([64, 256, 256, 8], 1024, True, None),      # cfg2 actor: one env step of all actors
    ([64, 256, 256, 8], 1000, True, None),      # rows not a multiple of the 16-row cluster tile
    ([17, 300, 200, 6], 333, True, None),       # reference default hidden sizes: odd K, n-tiles not a pass multiple
    ([33, 100, 52, 40], 50, False, None),       # wide LAST layer (written straight to global memory)
    ([10, 200, 120, 1], 77, False, (1, 4)),     # DDPG-critic shape: action concatenated into layer 1
    ([64, 300, 200, 8], 130, False, None),      # DDPG actor of configs[2]
    ([10, 44, 36, 3], 21, False, (1, 5)),       # aux columns sharing a k-step with the previous layer's tail
    ([12, 64, 5], 9, True, (0, 3)),             # aux on the input layer, 2-layer net
])
def test_mlp_forward_packed_matches_oracle(dims, rows, zf, aux):
    """Small-batch inference on pre-packed fragment-order weights (4-CTA cluster, resident weight slices, DSMEM)."""
    from surreal_b200 import ops
    gen = torch.Generator().manual_seed(sum(dims) + rows)
    aux_layer, aux_dim = aux if aux is not None else (-1, 0)
    layers = _rand_layers(dims, gen, aux_layer=aux_layer, aux_dim=aux_dim)
    acts = [ops.ACT_RELU] * (len(dims) - 2) + [ops.ACT_TANH if dims[-1] > 1 else ops.ACT_NONE]
    x = torch.randn(rows, dims[0], generator=gen) * 2 + 0.5
    a = torch.rand(rows, max(aux_dim, 1), generator=gen) * 2 - 1
    ozf, stats = None, None
    if zf:
        ozf = OZFilter(dims[0])
        ozf.update(torch.randn(200, dims[0], generator=gen) * 1.7 + 0.4)
        stats = torch.cat([ozf.running_sum, ozf.running_sumsq, ozf.count]).to(_dev())
    net = ops.FlatNet(dims, acts, _dev(), aux_layer=aux_layer, aux_dim=aux_dim).load_layers(layers)
    pk = ops.PackedWeights(net)
    assert pk.supported
    pk.refresh()
    out = ops.mlp_forward_packed(pk, x.to(_dev()), zf_stats=stats, aux=a.to(_dev()) if aux is not None else None)
    torch.cuda.synchronize()
    with torch.no_grad():
        h = ozf.forward(x) if zf else x
        for l, (w, b) in enumerate(layers):
            if l == aux_layer:
                h = torch.cat([h, a], 1)
            h = torch.nn.functional.linear(h, w, b)
            h = torch.relu(h) if acts[l] == ops.ACT_RELU else (torch.tanh(h) if acts[l] == ops.ACT_TANH else h)
    assert out.shape == h.shape
    assert_close_scale(out, h, 1e-5, 'packed forward')
    # a re-pack after a parameter change is picked up; an architecture with a narrow hidden layer is declined
    net.params.mul_(0.5)
    pk.refresh()
    out2 = ops.mlp_forward_packed(pk, x.to(_dev()), zf_stats=stats, aux=a.to(_dev()) if aux is not None else None)
    ref2 = ops.mlp_forward(net, x.to(_dev()), zf_stats=stats, aux=a.to(_dev()) if aux is not None else None)
    assert_close_scale(out2, ref2, 1e-5, 'packed vs tiled after re-pack')
    assert not ops.PackedWeights(ops.FlatNet([8, 16, 64, 2], [ops.ACT_RELU] * 3, _dev())).supported
    # a weight slice that does not fit one SM's shared memory is declined too (callers use the tiled forward)
    assert not ops.PackedWeights(ops.FlatNet([64, 1024, 1024, 8], [ops.ACT_RELU] * 3, _dev())).supported


def test_mlp_forward_dual_pipe_matches_single():
    """Large-batch forward split over the tensor pipe (3xTF32 mma tiles) and the FMA pipe (FFMA tiles) on two
    streams: same values as the default dispatch to fp32 rounding, every row written exactly once."""
    from surreal_b200 import ops
    gen = torch.Generator().manual_seed(11)
    dims, rows = [64, 256, 256, 1], 40000 + 37
    net = ops.FlatNet(dims, [ops.ACT_RELU, ops.ACT_RELU, ops.ACT_NONE], _dev()).load_layers(_rand_layers(dims, gen))
    x = (torch.randn(rows, 64, generator=gen) * 1.5).to(_dev())
    ozf = OZFilter(64)
    ozf.update(torch.randn(300, 64, generator=gen) * 1.7 + 0.4)
    stats = torch.cat([ozf.running_sum, ozf.running_sumsq, ozf.count]).to(_dev())
    ref = ops.mlp_forward(net, x, zf_stats=stats)
    for frac in (0.5, 0.3):
        out = torch.full((rows, 1), float('nan'), device=_dev())
        ops.mlp_forward_dual(net, x, zf_stats=stats, out=out, frac=frac)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(out).all())
        assert_close_scale(out, ref, 1e-5, 'dual-pipe forward, frac %.1f' % frac)
    for v in (1, 2):
        assert_close_scale(ops.mlp_forward(net, x, zf_stats=stats, variant=v), ref, 1e-5, 'variant %d' % v)


def test_mlp_forward_window_rows_and_aux():
    """virtual cat([obs, obs_next]) row mapping (ppo.py:376-383) and the DDPG critic's cat(h, action)."""
    from surreal_b200 import ops
    gen = torch.Generator().manual_seed(3)
    B, n, D, A = 13, 7, 10, 4
    layers = _rand_layers([D, 48, 36, 1], gen)
    obs = torch.randn(B, n, D, generator=gen)
    obs_next = torch.randn(B, 1, D, generator=gen)
    net = ops.FlatNet([D, 48, 36, 1], [ops.ACT_RELU, ops.ACT_RELU, ops.ACT_NONE], _dev()).load_layers(layers)
    out = ops.mlp_forward(net, obs.to(_dev()), x_next=obs_next.to(_dev()), win_n=n)
    with torch.no_grad():
        exp = onets.ppo_critic(torch.cat([obs, obs_next], 1).view(-1, D), layers)
    assert_close_scale(out, exp, 1e-5, 'window rows')

    layers = _rand_layers([D, 400, 300, 1], gen, aux_layer=1, aux_dim=A)
    x = torch.randn(77, D, generator=gen)
    act = torch.rand(77, A, generator=gen) * 2 - 1
    net = ops.FlatNet([D, 400, 300, 1], [ops.ACT_RELU, ops.ACT_RELU, ops.ACT_NONE], _dev(), aux_layer=1,
                      aux_dim=A).load_layers(layers)
    out = ops.mlp_forward(net, x.to(_dev()), aux=act.to(_dev()))
    with torch.no_grad():
        exp = onets.ddpg_critic(x, act, layers)
    assert_close_scale(out, exp, 1e-5, 'ddpg critic concat')


@pytest.mark.parametrize('tag', ['mlp', 'mlp_nonorm', 'rnn'])
def test_gae_matches_golden(golden, tag):
    from surreal_b200 import ops
    g = golden('gae_' + tag)
    r = torch.tensor(g['rewards'], dtype=torch.float32).to(_dev())
    v = torch.tensor(g['values_raw']).to(_dev())
    d = torch.tensor(g['dones']).to(_dev())
    H = int(g['horizon']) if 'horizon' in g else None
    adv, ret = ops.gae_window(r, v, d, float(g['gamma']), float(g['lam']), horizon=H, norm_adv=bool(g['norm_adv']))
    exp_adv, exp_ret = torch.tensor(g['adv']), torch.tensor(g['ret'])
    assert_close_scale(adv.view(-1), exp_adv.view(-1), 1e-5, 'adv')
    assert_close_scale(ret.view(-1), exp_ret.view(-1), 1e-5, 'ret')


@pytest.mark.parametrize('B,n,H,norm', [(1024, 128, None, True), (4096, 256, None, True), (64, 25, 5, True),
                                        (3, 1, None, False), (257, 33, 33, True), (40, 50, 7, False)])
def test_gae_matches_oracle(B, n, H, norm):
    from surreal_b200 import ops
    gen = torch.Generator().manual_seed(B + n)
    r = torch.randn(B, n, generator=gen) * 0.5
    v = torch.randn(B, n + 1, generator=gen)
    d = (torch.rand(B, n, generator=gen) < 0.05).float()
    adv, ret = ops.gae_window(r.to(_dev()), v.to(_dev()), d.to(_dev()), 0.995, 0.97, horizon=H, norm_adv=norm)
    e_adv, e_ret = gae_from_values(r, v, d, 0.995, 0.97, horizon=H, norm_adv=norm)
    tol = 1e-5
    if norm:   # normalised advantages: absolute 1e-5 (BASELINE.md §5)
        assert float((adv.cpu().view(-1) - e_adv.view(-1)).abs().max()) <= tol
    else:
        assert_close_scale(adv.view(-1), e_adv.view(-1), tol, 'adv')
    assert_close_scale(ret.view(-1), e_ret.view(-1), tol, 'ret')
    # a second call must reuse the (self-resetting) workspace correctly
    adv2, _ = ops.gae_window(r.to(_dev()), v.to(_dev()), d.to(_dev()), 0.995, 0.97, horizon=H, norm_adv=norm)
    assert torch.equal(adv, adv2)


@pytest.mark.parametrize('dims,rows,zf,win', [
    ([64, 256, 256, 1], 132096, True, 0),      # the cfg2 critic pass: 1032 tiles of 128 rows, 7-8 tiles per CTA
    ([64, 256, 256, 1], 128 * 5 + 77, True, 0),   # ragged last tile
    ([64, 256, 256, 8], 4096, True, 0),        # 8 output columns, tanh head
    ([32, 128, 64, 3], 19205, False, 0),       # narrower layers (one 128-column half each, layer 2 zero-padded), single layer-1 chunk
    ([128, 256, 256, 1], 1000, True, 0),       # four layer-1 chunks
    ([64, 256, 256, 1], 0, True, 16),          # virtual cat([obs, obs_next]) rows of ppo.py:376-383 (B = 600 windows)
])
def test_tcgen05_forward_matches_oracle(dims, rows, zf, win):
    """sb200_mlp_forward_tc5_f32 (wgmma tf32, accumulators in registers, 3xTF32 split) against the fp32 oracle
    network at 1e-5 * max(1, rms): same bar as the mma.sync / FFMA forward kernels."""
    from surreal_b200 import ops
    gen = torch.Generator().manual_seed(sum(dims) + rows + win)
    layers = _rand_layers(dims, gen)
    acts = [ops.ACT_RELU, ops.ACT_RELU, ops.ACT_TANH if dims[-1] > 1 else ops.ACT_NONE]
    D = dims[0]
    if win:
        B = 600
        xw = torch.randn(B, win, D, generator=gen) * 2 + 0.5
        xn = torch.randn(B, 1, D, generator=gen) * 2 + 0.5
        x = torch.cat([xw, xn], 1).reshape(-1, D)
        rows = x.shape[0]
    else:
        x = torch.randn(rows, D, generator=gen) * 2 + 0.5
    ozf, stats = None, None
    if zf:
        ozf = OZFilter(D)
        ozf.update(torch.randn(200, D, generator=gen) * 1.7 + 0.4)
        stats = torch.cat([ozf.running_sum, ozf.running_sumsq, ozf.count]).to(_dev())
    net = ops.FlatNet(dims, acts, _dev()).load_layers(layers)
    f = ops.Tc5Forward(net)
    assert f.supported(rows)
    out = torch.full((rows, dims[-1]), float('nan'), device=_dev())
    if win:
        f(xw.to(_dev()), out, zf_stats=stats, x_next=xn.to(_dev()), win_n=win)
    else:
        f(x.to(_dev()), out, zf_stats=stats)
    torch.cuda.synchronize()
    with torch.no_grad():
        h = ozf.forward(x) if zf else x
        for l, (w, b) in enumerate(layers):
            h = torch.nn.functional.linear(h, w, b)
            h = torch.relu(h) if acts[l] == ops.ACT_RELU else (torch.tanh(h) if acts[l] == ops.ACT_TANH else h)
    assert_close_scale(out, h, 1e-5, 'wgmma forward')
    # and the same rows through the default dispatcher (mma.sync / FFMA kernels) agree to the same bar
    ref = ops.mlp_forward(net, x.to(_dev()), zf_stats=stats)
    assert_close_scale(out, ref, 1e-5, 'wgmma vs default forward')

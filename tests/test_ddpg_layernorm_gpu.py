"""LayerNorm DDPG networks (model.use_layernorm) on the GPU: the forward epilogue of every dispatched kernel family and
the LayerNorm backward against float64, the per-actor forward, the entries that must reject a LayerNorm descriptor, and
DDPGLearner / DDPGAgent / checkpoints against goldens produced by the reference (make_golden_ddpg_layernorm.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import ddpg_configs, ref_state_dict
import ddpg_ln_ref as R
from test_ddpg_layernorm import LN_KEYS

pytestmark = pytest.mark.gpu
EPS = 1e-5


def _dev():
    return torch.device('cuda', 0)


def _net(dims, acts=None, aux_dim=0, seed=0, neg_bias0=False):
    from surreal_b200 import ops
    R = ops.ACT_RELU
    acts = acts or [R] * (len(dims) - 2) + [ops.ACT_TANH]
    net = ops.FlatNet(dims, acts, _dev(), aux_layer=1 if aux_dim else -1, aux_dim=aux_dim, layernorm=True)
    g = torch.Generator().manual_seed(seed)
    for l, lay in enumerate(net.layout):
        K, N = lay['K'], lay['N']
        b = (torch.rand(N, generator=g) - 0.5) * 0.2
        if neg_bias0 and l == 0:
            b = -0.05 - 0.1 * torch.rand(N, generator=g)
        net.set_layer(l, (torch.rand(N, K, generator=g) - 0.5) * (2.0 / K ** 0.5), b)
        if lay['g'] is not None:
            net.set_ln(l, 1.0 + 0.5 * torch.randn(N, generator=g), 0.3 * torch.randn(N, generator=g))
    return net


def _f64(net, x, aux=None):
    """float64 forward from the FlatNet's parameters: every layer's pre-LN activation and the output."""
    h = x.double().cpu()
    outs = []
    for l in range(net.n_layers):
        w, b = (t.double().cpu() for t in net.get_layer(l))
        if net.aux_layer == l:
            h = torch.cat([h, aux.double().cpu()], 1)
        h = h @ w.t() + b
        h = torch.relu(h) if net.acts[l] == 1 else (torch.tanh(h) if net.acts[l] == 2 else h)
        outs.append(h)
        if net.layout[l]['g'] is not None:
            gg, bb = (t.double().cpu() for t in net.get_ln(l))
            h = torch.nn.functional.layer_norm(h, h.shape[-1:], gg, bb, eps=EPS)
    return outs


def _ln64(h, g, b):
    return torch.nn.functional.layer_norm(h.double().cpu(), h.shape[-1:], g.double().cpu(), b.double().cpu(), eps=EPS)


NETS = [([17, 12, 20, 3], 0), ([33, 200, 300, 6], 0), ([40, 400, 300, 1], 6), ([9, 45, 13, 2], 3)]


@pytest.mark.parametrize('dims,aux', NETS)
@pytest.mark.parametrize('rows', [1, 5, 300, 2049, 4096, 6000])
@pytest.mark.parametrize('variant', [0, 1, 2, 'ffma'])
def test_forward_matches_float64(dims, aux, rows, variant):
    """Every kernel family: skinny (<= 2048 rows), mma tiles (variant 0 above 2048, variant 1), FFMA tiles (variant 2,
    and forward mode 0).  The LayerNorm epilogue against float64 of the kernel's own pre-LN rows, the output against a
    float64 forward.  Rows with x = 0 are all zero after the ReLU (negative first bias): their LayerNorm output is b."""
    from surreal_b200 import ops, _lib
    net = _net(dims, [1] * (len(dims) - 2) + [0 if aux else 2], aux_dim=aux, seed=rows, neg_bias0=True)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(rows, dims[0], generator=g)
    x[::7] = 0.0
    a = torch.rand(rows, aux, generator=g) * 2 - 1 if aux else None
    dev = _dev()
    xd, ad = x.to(dev), (a.to(dev) if aux else None)
    saves = [torch.zeros(rows, n, device=dev) for n in dims[1:]]
    lns = [torch.zeros(rows, n, device=dev) if net.layout[l]['g'] is not None else None for l, n in enumerate(dims[1:])]
    sts = [torch.zeros(rows, 2, device=dev) if t is not None else None for t in lns]
    if variant == 'ffma':
        _lib.lib().sb200_set_forward_mode(0)
    try:
        ops.mlp_forward(net, xd, aux=ad, saves=saves, ln_saves=lns, ln_stats=sts, variant=0 if variant == 'ffma' else variant)
        torch.cuda.synchronize()
    finally:
        _lib.lib().sb200_set_forward_mode(1)
    ref = _f64(net, x, a)
    for l in net.ln_layers():
        h = saves[l].cpu()
        gg, bb = (t.cpu() for t in net.get_ln(l))
        exp = _ln64(h, gg, bb)
        mean, rstd = h.double().mean(1, keepdim=True), 1.0 / (h.double().var(1, unbiased=False, keepdim=True) + EPS).sqrt()
        xhat = (h.double() - mean) * rstd
        tol = 4e-6 * (1.0 + mean.abs() * rstd + xhat.abs()) * gg.abs().max().double() + 1e-6
        assert bool(((lns[l].cpu().double() - exp).abs() <= tol).all()), ('LayerNorm epilogue', l)
        np.testing.assert_allclose(sts[l].cpu()[:, 0].numpy(), mean[:, 0].numpy(), rtol=1e-5, atol=1e-6)
        zero = (h == 0).all(1)
        assert int(zero.sum()) >= rows // 7 if l == 0 else True
        assert torch.equal(lns[l].cpu()[zero], bb.expand(int(zero.sum()), -1)), 'all-zero rows must give exactly b'
    out = saves[-1].cpu().double()
    scale = 1.0 + ref[-1].abs()
    assert float(((out - ref[-1]).abs() / scale).max()) <= 2e-4


@pytest.mark.parametrize('width', [12, 45, 300])
def test_forward_near_constant_rows(width):
    """Rows whose activations differ by ~1e-3 around 1: the variance is tiny and the two-pass reduction keeps it."""
    from surreal_b200 import ops
    net = _net([width, width, 4])
    net.set_layer(0, torch.eye(width), torch.zeros(width))
    g = torch.Generator().manual_seed(3)
    x = 1.0 + 1e-3 * torch.randn(64, width, generator=g)
    x[0] = 2.0                                                   # an exactly constant row: x^ = 0 -> b
    dev = _dev()
    saves = [torch.zeros(64, width, device=dev), torch.zeros(64, 4, device=dev)]
    ln = [torch.zeros(64, width, device=dev), None]
    ops.mlp_forward(net, x.to(dev), saves=saves, ln_saves=ln)
    h = saves[0].cpu()
    gg, bb = (t.cpu() for t in net.get_ln(0))
    exp = _ln64(h, gg, bb)
    tol = 2e-3 * gg.abs().max()                                 # fp32 mean of values near 1 over a std of 1e-3
    assert float((ln[0].cpu().double() - exp).abs().max()) <= tol
    assert torch.equal(ln[0].cpu()[0], bb)


@pytest.mark.parametrize('M,N,relu', [(1, 12, 1), (300, 45, 1), (4096, 400, 1), (1000, 300, 0)])
def test_backward_matches_float64(M, N, relu):
    from surreal_b200 import _lib, ops
    L = _lib.lib()
    g = torch.Generator().manual_seed(M + N)
    pre = torch.randn(M, N, generator=g)
    h = torch.relu(pre) if relu else pre
    h[::5] = 0.0 if relu else h[::5]
    gain, beta = 1.0 + 0.5 * torch.randn(N, generator=g), 0.3 * torch.randn(N, generator=g)
    dy = torch.randn(M, N, generator=g)
    mean = h.mean(1, keepdim=True)
    rstd = 1.0 / (h.var(1, unbiased=False, keepdim=True) + EPS).sqrt()
    stats = torch.cat([mean, rstd], 1).contiguous()
    dev = _dev()
    ld = ops._ru(N, 4)
    pad = lambda t: torch.nn.functional.pad(t, (0, ld - N)).contiguous().to(dev)  # noqa: E731
    hd, dyd, gd = pad(h), pad(dy), pad(gain.view(1, -1))[0].contiguous()
    dx = torch.zeros(M, ld, device=dev)
    splits, stride = 4, 3 * ld
    slabs = torch.full((splits, stride), 7.0, device=dev)
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    sd = stats.to(dev)
    ops.check(L.sb200_layernorm_bwd_f32(P(dyd), ld, P(hd), ld, P(sd), P(gd), M, N, relu, P(dx), ld,
                                        C.c_void_p(slabs.data_ptr()), C.c_void_p(slabs.data_ptr() + 4 * ld), stride,
                                        splits, ops._stream()), 'ln bwd')
    torch.cuda.synchronize()
    h64 = h.double().requires_grad_(True)
    g64, b64 = gain.double().requires_grad_(True), beta.double().requires_grad_(True)
    y = torch.nn.functional.layer_norm(h64, (N,), g64, b64, eps=EPS)
    y.backward(dy.double())
    dh = h64.grad * ((h > 0).double() if relu else 1.0)
    scale = float(dh.abs().max()) + 1e-6
    assert float((dx.cpu()[:, :N].double() - dh).abs().max()) <= 2e-5 * scale
    assert float(dx.cpu()[:, N:].abs().max() if ld > N else 0.0) == 0.0
    dg = slabs[:, :N].sum(0).cpu().double()
    db = slabs[:, ld:ld + N].sum(0).cpu().double()
    np.testing.assert_allclose(dg.numpy(), g64.grad.numpy(), rtol=0, atol=2e-5 * (1 + float(g64.grad.abs().max())))
    np.testing.assert_allclose(db.numpy(), b64.grad.numpy(), rtol=0, atol=2e-5 * (1 + float(b64.grad.abs().max())))
    assert bool((slabs[:, 2 * ld:] == 7.0).all()) and bool((slabs[:, N:ld] == 7.0).all())
    # no parameter gradient: the slabs stay untouched, dX is the same bits
    slabs.fill_(7.0)
    dx2 = torch.zeros_like(dx)
    ops.check(L.sb200_layernorm_bwd_f32(P(dyd), ld, P(hd), ld, P(sd), P(gd), M, N, relu, P(dx2), ld, None,
                                        None, stride, splits, ops._stream()), 'ln bwd')
    torch.cuda.synchronize()
    assert torch.equal(dx, dx2) and bool((slabs == 7.0).all())


@pytest.mark.parametrize('N', [1, 3, 1024])
def test_per_actor_forward_matches_float64(N):
    """Row k through image k (parameter noise) with LayerNorm, including the images' own gains and biases."""
    from surreal_b200 import ops, _lib
    dims = [33, 300, 200, 6]
    net = _net(dims, seed=1)
    stride = R.image_stride(dims)
    lay, size = R.flat_layout(dims)
    assert net.size == size and [(e['w'], e['b'], e['g'], e['beta']) for e in net.layout] == \
        [(e[0], e[1], e[5], e[6]) for e in lay]
    g = torch.Generator().manual_seed(N)
    imgs = net.params.cpu().repeat(N, 1)
    imgs = torch.nn.functional.pad(imgs, (0, stride - net.size)).contiguous()
    mask = torch.tensor(~R.padding_mask(dims, stride))
    imgs = imgs + 0.05 * torch.randn(imgs.shape, generator=g) * mask
    x = torch.randn(N, dims[0], generator=g)
    dev = _dev()
    im = imgs.reshape(-1).contiguous().to(dev)
    out = torch.zeros(N, dims[-1], device=dev)
    d = net.desc(im)
    xd = x.to(dev)
    ops.check(_lib.lib().sb200_mlp_forward_per_actor_f32(C.byref(d), stride, C.c_void_p(xd.data_ptr()), dims[0], N,
                                                         C.c_void_p(out.data_ptr()), dims[-1], None, None, 10, None,
                                                         ops._stream()), 'per actor')
    torch.cuda.synchronize()
    for k in range(N):
        net_k = net.clone_like()
        net_k.params.copy_(im[k * stride:k * stride + net.size])
        exp = _f64(net_k, x[k:k + 1])[-1]
        assert float((out[k].cpu().double() - exp[0]).abs().max()) <= 1e-5, k
        if k >= 4:
            break


def test_unsupported_entries_reject_layernorm():
    """Packed cluster forward, tc5 and the persistent rollout have no LayerNorm epilogue: they must say so."""
    from surreal_b200 import ops, _lib
    L = _lib.lib()
    for dims in ([64, 256, 256, 8], [32, 64, 64, 4]):
        net = _net(dims)
        plain = ops.FlatNet(dims, net.acts, _dev())
        d, dp = net.desc(), plain.desc()
        assert int(L.sb200_mlp_pack_floats(C.byref(d))) == 0
        assert not ops.PackedWeights(net).supported
        assert int(L.sb200_mlp_tc5_supported(C.byref(d), 4096)) == 0
        assert int(L.sb200_mlp_tc5_supported(C.byref(dp), 4096)) == int(dims[0] % 32 == 0)
        assert int(L.sb200_ppo_rollout_supported(C.byref(d), dims[0], dims[-1])) == 0
        buf = torch.zeros(1024, device=_dev())
        assert L.sb200_mlp_pack_tf32(C.byref(d), C.c_void_p(buf.data_ptr()), ops._stream()) == -3


def _learner(g, cfg, double):
    from surreal_b200.learner import DDPGLearner
    lc, ec, sc = ddpg_configs(D=cfg['D'], A=cfg['A'], actor_h=cfg['actor_h'], critic_h=cfg['critic_h'], B=cfg['B'],
                              n_step=cfg['n_step'], target=cfg['target'], clip_critic=cfg['clip_critic'],
                              lr_actor=cfg['lr_actor'], lr_critic=cfg['lr_critic'])
    lc.model.use_layernorm = True
    if double:
        lc.algo.network.use_double_critic = True
        lc.algo.network.use_action_regularization = bool(cfg['action_regularization'])
    L = DDPGLearner(lc, ec, sc)
    L.model.load_state_dict(ref_state_dict(g.sub('init/model/')))
    L.model_target.load_state_dict(ref_state_dict(g.sub('init/target/')))
    if double:
        L.model2.load_state_dict(ref_state_dict(g.sub('init/model2/')))
        L.model_target2.load_state_dict(ref_state_dict(g.sub('init/target2/')))
    return L


def _batch(b):
    return {'obs': {'low_dim': {'flat_inputs': b['obs']}}, 'obs_next': {'low_dim': {'flat_inputs': b['obs_next']}},
            'actions': b['actions'], 'rewards': b['rewards'], 'dones': b['dones']}


@pytest.mark.parametrize('tag', ['hard', 'soft_clipcritic', 'td3_double', 'td3_double_reg'])
def test_learner_matches_reference(golden, tag, monkeypatch):
    g = golden('ddpg_ln_optimize_' + tag)
    cfg, stats = g.js('cfg'), g.js('stats')
    double = tag.startswith('td3')
    runs = []
    for graph in ('1', '0'):
        monkeypatch.setenv('SB200_CUDA_GRAPH', graph)
        L = _learner(g, cfg, double)
        assert L.model.actor.ln_layers() == [0, 1] and L.model.critic.ln_layers() == [0, 1]
        assert not L.model.critic.layernorm or list(L.model.state_dict().keys()) == LN_KEYS
        for it in range(3):
            b = g.sub('it%d/' % it)
            if double and cfg['action_regularization']:
                L.policy_noise_draws = torch.tensor(b['policy_noise_unclipped'] / 0.2, dtype=torch.float32, device='cuda')
            st = L.learn(_batch(b))
            torch.cuda.synchronize()
            for k, v in stats[it].items():
                assert abs(st[k] - v) <= 1e-5 * max(1.0, abs(v)), '%s it%d: got %.9g expected %.9g' % (k, it, st[k], v)
            names = [('model', L.model), ('target', L.model_target)]
            if double:
                names += [('model2', L.model2), ('target2', L.model_target2)]
            for name, model in names:
                exp = ref_state_dict(g.sub('it%d/%s/' % (it, name)))
                got = model.state_dict()
                assert sorted(got) == sorted(exp)
                for k, e in exp.items():
                    d = float((got[k].cpu().reshape(e.shape) - e).abs().max())
                    assert d <= 2e-5, '%s %s it%d drift %.3e' % (name, k, it, d)      # lr_critic = 1e-3: 2% of one step
        runs.append([t.clone() for t in (L.model.actor.params, L.model.critic.params, L.model_target.critic.params,
                                         L.actor_optim.exp_avg, L.critic_optim.exp_avg_sq)])
    for a, b in zip(*runs):
        assert torch.equal(a, b), 'graph and eager learn() differ'


def test_out_of_range_actions_leave_state_untouched():
    from surreal_b200.learner import DDPGLearner
    lc, ec, sc = ddpg_configs(D=9, A=3, B=16, target={'type': 'soft', 'tau': 0.01, 'interval': 1})
    lc.model.use_layernorm = True
    L = DDPGLearner(lc, ec, sc)
    rng = np.random.default_rng(0)
    mk = lambda amax: {'obs': {'low_dim': {'flat_inputs': rng.standard_normal((16, 9)).astype(np.float32)}},   # noqa: E731
                       'obs_next': {'low_dim': {'flat_inputs': rng.standard_normal((16, 9)).astype(np.float32)}},
                       'actions': (rng.uniform(-1, 1, (16, 3)) * amax).astype(np.float32),
                       'rewards': rng.standard_normal((16, 1)), 'dones': np.zeros((16, 1))}
    L.learn(mk(1.0))
    snap = [t.clone() for t in (L.model.actor.params, L.model.critic.params, L.model_target.critic.params,
                                L.critic_optim.exp_avg_sq)]
    with pytest.raises(AssertionError):
        L.learn(mk(3.0))
    torch.cuda.synchronize()
    for a, b in zip(snap, (L.model.actor.params, L.model.critic.params, L.model_target.critic.params,
                           L.critic_optim.exp_avg_sq)):
        assert torch.equal(a, b)


def test_checkpoint_round_trip_continues_bit_identically(golden):
    from surreal_b200.learner import DDPGLearner
    g = golden('ddpg_ln_optimize_soft_clipcritic')
    cfg = g.js('cfg')
    L = _learner(g, cfg, False)
    L.session_config.checkpoint.learner.include_optimizer = True
    L.learn(_batch(g.sub('it0/')))
    attrs = L.checkpoint_attributes()
    assert 'critic_optim' in attrs and 'model_target' in attrs
    # what the checkpoint stores for every attribute (surreal_b200/checkpoint.py): state_dict() on the CPU, or the value
    data = {}
    for a in attrs:
        v = getattr(L, a)
        data[a] = {k: (t.detach().cpu().clone() if isinstance(t, torch.Tensor) else t) for k, t in v.state_dict().items()} \
            if hasattr(v, 'state_dict') else v
    lc, ec, sc = ddpg_configs(D=cfg['D'], A=cfg['A'], actor_h=cfg['actor_h'], critic_h=cfg['critic_h'], B=cfg['B'],
                              n_step=cfg['n_step'], target=cfg['target'], clip_critic=cfg['clip_critic'],
                              lr_actor=cfg['lr_actor'], lr_critic=cfg['lr_critic'])
    lc.model.use_layernorm = True
    L2 = DDPGLearner(lc, ec, sc)
    for a in attrs:
        cur = getattr(L2, a)
        if hasattr(cur, 'load_state_dict'):
            cur.load_state_dict(data[a])
        else:
            setattr(L2, a, data[a])
    assert list(L2.model.state_dict().keys()) == LN_KEYS
    for k, v in L.model.state_dict().items():
        assert tuple(v.shape) == tuple(g['init/model/' + k.replace('.', '/')].shape)
    for b in (g.sub('it1/'), g.sub('it2/')):
        s1, s2 = L.learn(_batch(b)), L2.learn(_batch(b))
        assert all(s1[k] == s2[k] for k in ('actor_loss', 'critic_loss', 'Q_policy'))
    for a, b in ((L.model.actor.params, L2.model.actor.params), (L.model.critic.params, L2.model.critic.params),
                 (L.model_target.critic.params, L2.model_target.critic.params)):
        assert torch.equal(a, b)


def test_agent_act_matches_reference(golden):
    from surreal_b200.agent import DDPGAgent
    g = golden('ddpg_ln_act')
    N = len(g['obs'])
    lc, ec, sc = ddpg_configs(D=9, A=3)
    lc.model.use_layernorm = True
    ec.num_envs, ec.num_agents = N, 4
    ag = DDPGAgent(lc, ec, sc, 0, 'training')
    assert not ag._packed.supported                          # the packed cluster forward has no LayerNorm
    ag.model.load_state_dict(ref_state_dict(g.sub('model/')))
    ag._sigma.fill_(float(g['sigma']))
    a = ag.act({'low_dim': {'flat_inputs': torch.tensor(g['obs'], device=_dev())}}, unit_noise=g['unit_noise'])
    np.testing.assert_allclose(a.cpu().numpy(), g['actions'], rtol=0, atol=2e-6)
    a = ag.act({'low_dim': {'flat_inputs': g['obs']}}, unit_noise=g['unit_noise'])      # host observations
    np.testing.assert_allclose(a, g['actions'], rtol=0, atol=2e-6)


def test_agent_ou_noise_matches_reference(golden):
    from surreal_b200.agent import DDPGAgent
    g = golden('ddpg_ln_act_ou')
    lc, ec, sc = ddpg_configs(D=9, A=3)
    lc.model.use_layernorm = True
    lc.algo.exploration.noise_type = 'ou_noise'
    lc.algo.exploration.theta, lc.algo.exploration.dt = float(g['theta']), float(g['dt'])
    ec.num_envs, ec.num_agents = 1, 4
    ag = DDPGAgent(lc, ec, sc, 0, 'training')
    ag.model.load_state_dict(ref_state_dict(g.sub('model/')))
    ag._sigma64.fill_(float(g['sigma']))
    for i in range(len(g['obs'])):
        if i == int(g['reset_at']):
            ag.pre_episode()
        a = ag.act({'low_dim': {'flat_inputs': g['obs'][i:i + 1]}}, unit_noise=g['unit_noise'][i:i + 1])
        np.testing.assert_allclose(a[0], g['actions'][i], rtol=0, atol=2e-6)
        np.testing.assert_allclose(ag._ou_state.cpu().numpy()[0], g['ou_states'][i], rtol=0, atol=1e-7)


def _actor_entries(sd, pre):
    return [(sd[pre + 'seq/%d/weight' % (3 * l)], sd[pre + 'seq/%d/bias' % (3 * l)]) +
            ((sd[pre + 'seq/%d/weight' % (3 * l + 2)], sd[pre + 'seq/%d/bias' % (3 * l + 2)]) if l < 2 else ())
            for l in range(3)]


@pytest.mark.parametrize('tag', ['normal', 'adaptive'])
@pytest.mark.parametrize('host', [False, True])
def test_param_noise_agent_matches_reference(golden, tag, host):
    """Actor k of DDPGAgent(num_envs=3) replays reference agent k with the injected draws: perturbed images (LayerNorm
    gains and biases included) exact, sigma exact, actions <= 2e-6."""
    from surreal_b200.agent import DDPGAgent
    g = golden('ddpg_ln_param_noise_' + tag)
    cfg = g.js('cfg')
    lc, ec, sc = ddpg_configs(D=9, A=3)
    lc.model.use_layernorm = True
    ex = lc.algo.exploration
    ex.param_noise_type = cfg['kind']
    ex.param_noise_sigma, ex.param_noise_alpha = cfg['sigma'], cfg['alpha']
    ec.num_envs, ec.num_agents = 3, 3
    ag = DDPGAgent(lc, ec, sc, 0, 'training')
    ag.param_noise_target_stddev = cfg['target_stddev']
    dims = [cfg['D']] + cfg['actor_h'] + [cfg['A']]
    stride = ag.param_noise_stride
    assert stride == R.image_stride(dims)
    for f in range(cfg['fetches']):
        for l, e in enumerate(_actor_entries(g.sub('f%d/model/' % f), 'actor/model/')):
            ag.model.actor.set_layer(l, torch.tensor(e[0]), torch.tensor(e[1]))
            if len(e) == 4:
                ag.model.actor.set_ln(l, torch.tensor(e[2]), torch.tensor(e[3]))
        un = np.stack([R.to_flat(_actor_entries(g.sub('a%d/f%d/pz/' % (k, f)), 'actor/model/'), dims, stride,
                                  dtype=np.float64) for k in range(3)])
        ag.apply_param_noise(unit_noise=un)
        assert ag.param_noise_sigma.tolist() == [float(g['a%d/sigma' % k][f]) for k in range(3)]
        imgs = ag._pn_images.view(3, stride).cpu().numpy()
        for k in range(3):
            exp = R.to_flat(_actor_entries(g.sub('a%d/f%d/pert/' % (k, f)), 'actor/model/'), dims, stride)
            np.testing.assert_array_equal(imgs[k], exp)
        for t in range(cfg['acts']):
            obs = np.stack([g['obs'][f, t]] * 3)
            un_a = np.stack([g['a%d/action_z' % k][f, t] for k in range(3)])
            a = ag.act(obs if host else torch.tensor(obs, device=_dev()), unit_noise=un_a)
            a = a if host else a.cpu().numpy()
            for k in range(3):
                np.testing.assert_allclose(a[k], g['a%d/actions' % k][f, t], rtol=0, atol=2e-6)


@pytest.mark.parametrize('param_noise', [None, 'adaptive_normal'])
def test_launcher_end_to_end(param_noise):
    """actors -> n-step SSAR staging -> UniformReplay -> DDPGLearner with use_layernorm=True, with and without
    parameter noise (device env, graph-captured chunks where the agent uses them)."""
    from surreal_b200.launch import SurrealDefaultLauncher
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.learner import DDPGLearner
    from surreal_b200.replay import UniformReplay
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    N = 16
    lc, ec, sc = ddpg_configs(D=12, A=4, actor_h=(48, 32), critic_h=(64, 48), B=64, n_step=3, memory_size=500, start=100)
    lc.model.use_layernorm = True
    lc.algo.exploration.param_noise_type = param_noise
    make_synthetic_env_config(ec, N, 12, 4, seed=1)
    ec.num_agents = N
    ec.limit_episode_length = 20
    la = SurrealDefaultLauncher(DDPGAgent, DDPGLearner, UniformReplay, sc, ec, lc)
    agent, replay, learner = la.setup_engine()
    assert agent.model.actor.layernorm and learner.model.critic.layernorm
    agent.main_loop(max_steps=30)
    torch.cuda.synchronize()
    assert len(replay) == N * (18 + (30 - 20 - 2))
    st = learner.learn(replay.sample(64))
    assert all(np.isfinite(st[k]) for k in ('actor_loss', 'critic_loss', 'Q_policy'))
    assert float(replay.r_act.abs().max()) <= 1.0

"""DDPG parameter-space noise on the GPU: the perturbation kernel (Philox stream, injected draws, padding), the per-actor
forward against float64, the agent against the reference goldens, and the device-chunk / eager / host paths."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from helpers import ddpg_configs
from oracle import param_noise as PN

pytestmark = pytest.mark.gpu

R, T = 1, 2           # ACT_RELU, ACT_TANH


def _dev():
    return torch.device('cuda', 0)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _net(dims, seed=0, scale=None):
    from surreal_b200 import ops
    net = ops.FlatNet(dims, [R] * (len(dims) - 2) + [T], _dev())
    g = torch.Generator().manual_seed(seed)
    layers = [((torch.rand(dims[l + 1], dims[l], generator=g) * 2 - 1) * (scale or dims[l] ** -0.5),
               (torch.rand(dims[l + 1], generator=g) * 2 - 1) * 0.1) for l in range(len(dims) - 1)]
    return net.load_layers(layers)


def _apply(net, N, images, stride, sigma, unit=None, seed=5, fetch=0, dist=None, state=None, alpha=1.15, target=0.005):
    from surreal_b200 import _lib, ops
    d = net.desc()
    _lib.check(_lib.lib().sb200_ddpg_param_noise_apply_f32(C.byref(d), N, _p(images), stride, _p(sigma), _p(unit), seed,
                                                           fetch, _p(dist), _p(state), alpha, target, ops._stream()),
               'apply')


def _forward(net, images, stride, x, out, shared=None, dist=None, state=None):
    from surreal_b200 import _lib, ops
    d = net.desc(images) if images is not None else net.desc()
    s = shared.desc() if shared is not None else None
    _lib.check(_lib.lib().sb200_mlp_forward_per_actor_f32(
        C.byref(d), stride, _p(x), x.stride(0), x.shape[0], _p(out), out.stride(0), C.byref(s) if s is not None else None,
        _p(dist), 10, _p(state), ops._stream()), 'forward')
    return out


# -- 1. perturbation --------------------------------------------------------------------------------------------------
def test_philox_draws_match_oracle():
    """W = 0, sigma = 1: each image is fl32(z) of the device's double Box-Muller draws, equal to the oracle's stream."""
    dims = [17, 48, 32, 3]
    net = _net(dims)
    net.params.zero_()
    N, stride = 4, PN.image_stride(dims)
    images = torch.full((N * stride,), 7.0, device=_dev())
    sigma = torch.ones(N, dtype=torch.float64, device=_dev())
    pad = PN.padding_mask(dims, stride)
    for fetch in (0, 3):
        _apply(net, N, images, stride, sigma, seed=123, fetch=fetch)
        got = images.view(N, stride).cpu().numpy()
        for k in range(N):
            exp = PN.param_noise_unit(123, fetch, k, stride).astype(np.float32)
            exp[pad] = 0.0
            np.testing.assert_array_equal(got[k], exp)
        assert np.all(got[:, pad] == 0.0)
        assert len({got[k].tobytes() for k in range(N)}) == N            # distinct per actor
    first = images.clone()
    _apply(net, N, images, stride, sigma, seed=123, fetch=1)
    assert not torch.equal(first, images)                                    # distinct per fetch


def test_injected_draws_give_numpy_rounding():
    dims = [9, 20, 12, 3]
    net = _net(dims, seed=1)
    N, stride = 5, PN.image_stride(dims)
    rng = np.random.default_rng(0)
    z = rng.standard_normal((N, stride))
    sig = np.array([0.05, 0.3, 1e-3, 2.0, 0.0])
    images = torch.full((N * stride,), -1.0, device=_dev())
    _apply(net, N, images, stride, torch.tensor(sig, device=_dev()), unit=torch.tensor(z, device=_dev()))
    W = net.params.cpu().numpy()
    flat = np.zeros(stride, np.float32)
    flat[:W.size] = W
    pad = PN.padding_mask(dims, stride)
    got = images.view(N, stride).cpu().numpy()
    for k in range(N):
        exp = (flat.astype(np.float64) + sig[k] * z[k]).astype(np.float32)
        exp[pad] = 0.0
        np.testing.assert_array_equal(got[k], exp)


def test_adaptive_apply_updates_sigma_on_device():
    """dist / i in float32 against the target; /= alpha above it, *= alpha otherwise; skipped at i = 0; i reset."""
    dims = [5, 8, 2]
    net = _net(dims)
    N, stride = 4, PN.image_stride(dims)
    images = torch.zeros(N * stride, device=_dev())
    sigma = torch.full((N,), 0.05, dtype=torch.float64, device=_dev())
    dist = torch.tensor([0.0, 0.1, 0.23, 0.2300001], device=_dev())
    state = torch.zeros(2, dtype=torch.int64, device=_dev())
    _apply(net, N, images, stride, sigma, dist=dist, state=state, alpha=1.15, target=0.01)
    assert sigma.cpu().tolist() == [0.05] * 4 and int(state[0]) == 0       # i == 0: nothing to adapt
    state[0] = 23
    _apply(net, N, images, stride, sigma, dist=dist, state=state, alpha=1.15, target=0.01)
    d32 = dist.cpu().numpy()
    exp = []
    for k in range(N):
        mean = torch.tensor(d32[k]) / 23
        exp.append(0.05 / 1.15 if bool(mean > 0.01) else 0.05 * 1.15)
    assert sigma.cpu().tolist() == exp and int(state[0]) == 0


# -- 2. per-actor forward ---------------------------------------------------------------------------------------------
NETS = [[64, 300, 200, 8], [17, 48, 32, 3], [13, 37, 1]]


def _f64_forward(imgs, dims, x):
    """imgs [N][stride] float32 -> float64 per-actor forward."""
    h = x.double()
    lay, _ = PN.flat_layout(dims)
    for l, (w_off, b_off, K, Nn, ldw) in enumerate(lay):
        W = imgs[:, w_off:w_off + K * ldw].double().view(-1, K, ldw)[:, :, :Nn]
        b = imgs[:, b_off:b_off + Nn].double()
        h = torch.bmm(h.unsqueeze(1), W).squeeze(1) + b
        h = torch.tanh(h) if l == len(lay) - 1 else torch.relu(h)
    return h


@pytest.mark.parametrize('dims', NETS)
@pytest.mark.parametrize('N', [1, 3, 131, 1024, 4096])
def test_per_actor_forward_matches_float64(dims, N):
    net = _net(dims, seed=N)
    stride = PN.image_stride(dims)
    g = torch.Generator(device=_dev()).manual_seed(N)
    images = torch.zeros(N, stride, device=_dev())
    base = torch.zeros(stride, device=_dev())
    base[:net.size] = net.params
    mask = torch.tensor(~PN.padding_mask(dims, stride), device=_dev())
    images[:] = (base + 0.05 * torch.randn(N, stride, device=_dev(), generator=g)) * mask
    x = torch.randn(N, dims[0], device=_dev(), generator=g)
    out = torch.full((N, dims[-1]), float('nan'), device=_dev())
    _forward(net, images, stride, x, out)
    ref = _f64_forward(images, dims, x)
    # output scale, floored at 1e-2: a lone row whose tanh output sits near 0 keeps the fp32 rounding of its hidden layers
    scale = max(float(ref.abs().max()), 1e-2)
    err = float((out.double() - ref).abs().max())
    assert err <= 1e-5 * scale, err
    out2 = torch.empty_like(out)
    _forward(net, images, stride, x, out2)
    assert torch.equal(out, out2)                                            # fixed-order sums
    del images, ref


@pytest.mark.parametrize('dims', NETS)
def test_shared_images_match_mlp_forward(dims):
    from surreal_b200 import ops
    net = _net(dims, seed=3)
    N = 257
    x = torch.randn(N, dims[0], device=_dev())
    out = torch.empty(N, dims[-1], device=_dev())
    _forward(net, None, 0, x, out)                                           # stride 0: every row reads net.params
    ref = ops.mlp_forward(net, x)
    assert float((out - ref).abs().max()) <= 2e-6


@pytest.mark.parametrize('dims', NETS[:2])
def test_adaptive_distance_matches_float64(dims):
    net = _net(dims, seed=4)
    N, stride = 131, PN.image_stride(dims)
    mask = torch.tensor(~PN.padding_mask(dims, stride), device=_dev())
    base = torch.zeros(stride, device=_dev())
    base[:net.size] = net.params
    images = (base + 0.02 * torch.randn(N, stride, device=_dev())) * mask
    x = torch.randn(N, dims[0], device=_dev())
    out = torch.empty(N, dims[-1], device=_dev())
    dist = torch.full((N,), -1.0, device=_dev())
    state = torch.zeros(2, dtype=torch.int64, device=_dev())
    _forward(net, images, stride, x, out, shared=net, dist=dist, state=state)
    ref = (_f64_forward(images, dims, x) - _f64_forward(base.unsqueeze(0).expand(N, -1), dims, x)).pow(2).sum(1).sqrt()
    assert float((dist.double() - ref).abs().max()) <= 1e-5 * max(float(ref.max()), 1e-3)
    assert int(state[0]) == 1 and int(state[1]) == 0
    dist.fill_(-1.0)
    for _ in range(9):                                                       # acts 1..9: no distance
        _forward(net, images, stride, x, out, shared=net, dist=dist, state=state)
    assert bool((dist == -1.0).all()) and int(state[0]) == 10
    _forward(net, images, stride, x, out, shared=net, dist=dist, state=state)   # act 10 measures again
    assert bool((dist >= 0).all()) and int(state[0]) == 11


# -- 3. the agent against the reference -------------------------------------------------------------------------------
def _agent(kind, N=3, mode='training', **kw):
    from surreal_b200.agent import DDPGAgent
    lc, ec, sc = ddpg_configs(D=9, A=3, **kw)
    ex = lc.algo.exploration
    ex.param_noise_type = kind
    ex.param_noise_sigma, ex.param_noise_alpha = 0.05, 1.15
    ec.num_envs, ec.num_agents = N, N
    return DDPGAgent(lc, ec, sc, 0, mode), (lc, ec, sc)


def _set_actor(ag, sd):
    for l in range(ag.model.actor.n_layers):
        ag.model.actor.set_layer(l, torch.tensor(sd['actor/model/seq/%d/weight' % (2 * l)]),
                                 torch.tensor(sd['actor/model/seq/%d/bias' % (2 * l)]))


@pytest.mark.parametrize('tag', ['normal', 'adaptive'])
@pytest.mark.parametrize('host', [False, True])
def test_agent_matches_reference(golden, tag, host):
    """Actor k of DDPGAgent(num_envs=3) replays reference agent k: perturbed weights, sigma trajectory, actions."""
    g = golden('ddpg_param_noise_' + tag)
    cfg = g.js('cfg')
    kind = cfg['kind']
    ag, _ = _agent(kind)
    ag.param_noise_target_stddev = cfg['target_stddev']
    dims = [cfg['D']] + cfg['actor_h'] + [cfg['A']]
    stride = ag.param_noise_stride
    assert stride == PN.image_stride(dims)
    np.testing.assert_array_equal(ag.sigma, [float(g['a%d/action_sigma' % k]) for k in range(3)])
    for f in range(cfg['fetches']):
        _set_actor(ag, g.sub('f%d/model/' % f))
        un = np.stack([PN.to_flat([(g['a%d/f%d/pz/actor/model/seq/%d/weight' % (k, f, 2 * l)],
                                    g['a%d/f%d/pz/actor/model/seq/%d/bias' % (k, f, 2 * l)]) for l in range(len(dims) - 1)],
                                  dims, stride, dtype=np.float64) for k in range(3)])
        ag.apply_param_noise(unit_noise=un)
        assert ag.param_noise_sigma.tolist() == [float(g['a%d/sigma' % k][f]) for k in range(3)]
        imgs = ag._pn_images.view(3, stride).cpu().numpy()
        for k in range(3):
            exp = PN.to_flat([(g['a%d/f%d/pert/actor/model/seq/%d/weight' % (k, f, 2 * l)],
                               g['a%d/f%d/pert/actor/model/seq/%d/bias' % (k, f, 2 * l)]) for l in range(len(dims) - 1)],
                             dims, stride)
            np.testing.assert_array_equal(imgs[k], exp)
        for t in range(cfg['acts']):
            obs = np.stack([g['obs'][f, t]] * 3)
            un_a = np.stack([g['a%d/action_z' % k][f, t] for k in range(3)])
            a = ag.act(obs if host else torch.tensor(obs, device=_dev()), unit_noise=un_a)
            a = a if host else a.cpu().numpy()
            for k in range(3):
                np.testing.assert_allclose(a[k], g['a%d/actions' % k][f, t], rtol=0, atol=2e-6)


def test_eval_deterministic_uses_unperturbed_weights():
    from surreal_b200 import ops
    ag, _ = _agent('normal', N=4, mode='eval_deterministic')
    assert ag.param_noise_type is None and ag.param_noise_sigma is None
    x = torch.randn(4, 9, device=_dev())
    a = ag.act(x).clone()
    ref = ops.mlp_forward(ag.model.actor, x).clamp(-1, 1)
    assert torch.equal(a, ref)


def test_fetch_loads_snapshot_then_perturbs():
    """fetch_parameter -> on_parameter_fetched: the model holds the unperturbed snapshot, the images its perturbation."""
    from surreal_b200.distributed import LocalHub, ParameterPublisher
    ag, (lc, ec, sc) = _agent('adaptive_normal', N=5)
    src, _ = _agent('adaptive_normal', N=5)
    src.model.actor.params.mul_(1.5)
    pub = ParameterPublisher({'ddpg': src.model})
    LocalHub.get(sc).publisher = pub
    pub.publish(0)
    ag.fetch_parameter()
    assert torch.equal(ag.model.actor.params, src.model.actor.params)
    stride = ag.param_noise_stride
    imgs = ag._pn_images.view(5, stride)
    n = ag.model.actor.size
    diff = (imgs[:, :n] - ag.model.actor.params).abs()
    assert float(diff.max()) > 0 and float(diff.max()) < 1.0
    ag.fetch_parameter()                                        # same version: no new draws (the client returns None)
    assert torch.equal(imgs, ag._pn_images.view(5, stride))
    assert ag._pn_fetches == 1


# -- 4. device chunk (graph / eager) and host loop agree -------------------------------------------------------------
@pytest.mark.parametrize('kind', ['normal', 'adaptive_normal'])
def test_device_chunk_graph_equals_eager(monkeypatch, kind):
    from surreal_b200.env import SyntheticEnv
    from surreal_b200.replay import UniformReplay
    runs = []
    N, D, A = 37, 12, 4
    for graphs in ('1', '0'):
        monkeypatch.setenv('SB200_CUDA_GRAPH', graphs)
        from surreal_b200.agent import DDPGAgent
        lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=(48, 32), critic_h=(64, 48), n_step=3, memory_size=400, start=0)
        lc.algo.exploration.param_noise_type = kind
        ec.num_envs, ec.num_agents = N, N
        ec.limit_episode_length = 9
        R = UniformReplay(lc, ec, sc)
        torch.manual_seed(3)
        ag = DDPGAgent(lc, ec, sc, 0, 'training')
        ag.model.actor.params.mul_(3.0)
        ag.main_setup(SyntheticEnv(N, D, A, 9, seed=4))
        sigmas = []
        for chunk in range(4):
            if chunk in (1, 3):
                ag.apply_param_noise()                          # a fetch between chunks
                sigmas.append(ag.param_noise_sigma.tolist())
            ag.main_loop(max_steps=6)
        torch.cuda.synchronize()
        runs.append(dict(n=len(R), sig=sigmas, img=ag._pn_images.clone(),
                         ring=[x.clone() for x in (R.r_obs, R.r_obs_next, R.r_act, R.r_rew, R.r_done)]))
    a, b = runs
    assert a['n'] == b['n'] > 0 and a['sig'] == b['sig']
    assert torch.equal(a['img'], b['img'])
    for x, y in zip(a['ring'], b['ring']):
        assert torch.equal(x, y)


@pytest.mark.parametrize('kind', ['normal', 'adaptive_normal'])
@pytest.mark.parametrize('noise', ['normal', 'ou_noise'])
def test_host_env_equals_device_env(kind, noise):
    from test_host_env_gpu import Stream, NumpyEnv, TorchEnv
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.replay import UniformReplay
    N, D, A, Tn = 9, 12, 4, 30
    s = Stream(N, D, Tn, seed=7)
    runs, sd = [], None
    for host in (True, False):
        lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=(48, 32), critic_h=(64, 48), n_step=3, memory_size=100, start=0)
        lc.algo.exploration.noise_type = noise
        lc.algo.exploration.param_noise_type = kind
        ec.num_envs = N
        R = UniformReplay(lc, ec, sc)
        ag = DDPGAgent(lc, ec, sc, 0, 'training')
        if sd is None:
            sd = {k: v.clone() for k, v in ag.model.state_dict().items()}
        else:
            ag.model.load_state_dict(sd)
        ag.env = w = ag.prepare_env_agent(NumpyEnv(s, A, rew64=True) if host else TorchEnv(s, A))
        obs, _ = w.reset()
        acts = []
        for t in range(Tn):
            if t % 11 == 3:
                ag.apply_param_noise()
            a = ag.act(obs)
            acts.append(torch.from_numpy(a.copy()) if host else a.cpu().clone())
            obs, _, _, _ = w.step(a)
        torch.cuda.synchronize()
        runs.append(dict(acts=acts, sig=ag.param_noise_sigma.tolist(),
                         ring=[x.clone() for x in (R.r_obs, R.r_obs_next, R.r_act, R.r_rew, R.r_done)]))
    h, d = runs
    for t in range(Tn):
        assert torch.equal(h['acts'][t], d['acts'][t]), t
    assert h['sig'] == d['sig']
    for x, y in zip(h['ring'], d['ring']):
        assert torch.equal(x, y)

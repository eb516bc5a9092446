"""LayerNorm DDPG networks (model.use_layernorm) without a GPU: the CPU restatement (tests/ddpg_ln_ref.py, on top of
oracle/) against goldens produced by the reference with use_layernorm=True (tests/golden/make_golden_ddpg_layernorm.py)."""
import numpy as np
import pytest
import torch

import ddpg_ln_ref as R
from ddpg_ln_ref import actor_layers, critic_layers, ddpg_act, ddpg_act_ou
from oracle import param_noise as PN

# the reference's state-dict keys with use_layernorm (Linear, ReLU, LayerNorm per hidden layer)
LN_KEYS = ['actor.model.seq.%d.%s' % (i, p) for i in (0, 2, 3, 5, 6) for p in ('weight', 'bias')] + \
          ['critic.model_obs.seq.%d.%s' % (i, p) for i in (0, 2) for p in ('weight', 'bias')] + \
          ['critic.model_concat.seq.%d.%s' % (i, p) for i in (0, 2, 3) for p in ('weight', 'bias')]


def test_fixture_keys_are_the_reference_layout(golden):
    g = golden('ddpg_ln_optimize_hard')
    keys = sorted(k.replace('/', '.') for k in g.sub('init/model/'))
    assert keys == sorted(LN_KEYS)
    sd = g.sub('init/model/')
    assert sd['actor/model/seq/2/weight'].shape == (20,) and sd['critic/model_concat/seq/2/bias'].shape == (16,)


def test_layernorm_matches_torch_module():
    """F.layer_norm with eps 1e-5 and (gain, bias) is what torch.nn.LayerNorm(width) computes."""
    torch.manual_seed(0)
    ln = torch.nn.LayerNorm(13)
    with torch.no_grad():
        ln.weight.add_(torch.randn(13))
        ln.bias.add_(torch.randn(13))
    x = torch.randn(7, 13)
    e = (torch.eye(13), torch.zeros(13), ln.weight.detach(), ln.bias.detach())     # identity Linear: exact
    assert ln.eps == R.LAYERNORM_EPS
    with torch.no_grad():
        assert torch.equal(R.hidden(x, e), ln(torch.relu(x)))


@pytest.mark.parametrize('tag', ['hard', 'soft_clipcritic', 'td3_double', 'td3_double_reg'])
def test_oracle_optimize_matches_reference(golden, tag):
    g = golden('ddpg_ln_optimize_' + tag)
    cfg = g.js('cfg')
    double = tag.startswith('td3')
    kw = dict(gamma=cfg['gamma'], n_step=cfg['n_step'], lr_actor=cfg['lr_actor'], lr_critic=cfg['lr_critic'],
              clip_actor=cfg['clip_actor'], actor_clip=cfg['actor_clip'], clip_critic=cfg['clip_critic'],
              critic_clip=cfg['critic_clip'], target_type=cfg['target']['type'],
              target_interval=cfg['target'].get('interval', 0), tau=cfg['target'].get('tau', 0.0))
    if double:
        kw.update(critic2=critic_layers(g.sub('init/model2/')), critic2_t=critic_layers(g.sub('init/target2/')))
    L = R.LayerNormDDPGLearner(actor_layers(g.sub('init/model/')), critic_layers(g.sub('init/model/')),
                          actor_layers(g.sub('init/target/')), critic_layers(g.sub('init/target/')), **kw)
    stats = g.js('stats')
    for it in range(3):
        b = g.sub('it%d/' % it)
        noise = b['policy_noise_unclipped'] if double and cfg['action_regularization'] else None
        st = L.optimize(b['obs'], b['actions'], b['rewards'], b['obs_next'], b['dones'], policy_noise=noise)
        for k, v in stats[it].items():
            assert st[k] == pytest.approx(v, rel=1e-6, abs=1e-7), k
        pairs = [(L.actor, actor_layers(g.sub('it%d/model/' % it))), (L.critic, critic_layers(g.sub('it%d/model/' % it))),
                 (L.actor_t, actor_layers(g.sub('it%d/target/' % it))),
                 (L.critic_t, critic_layers(g.sub('it%d/target/' % it)))]
        if double:
            pairs += [(L.critic2, critic_layers(g.sub('it%d/model2/' % it))),
                      (L.critic2_t, critic_layers(g.sub('it%d/target2/' % it)))]
        for got, exp in pairs:
            for eg, ee in zip(got, exp):
                assert len(eg) == len(ee)
                for t, e in zip(eg, ee):
                    np.testing.assert_allclose(t.detach().numpy(), e.numpy(), rtol=0, atol=1e-7)


def test_oracle_act_matches_reference(golden):
    g = golden('ddpg_ln_act')
    actor = actor_layers(g.sub('model/'))
    for i in range(len(g['obs'])):
        a = ddpg_act(g['obs'][i], actor, float(g['sigma']), g['unit_noise'][i])
        np.testing.assert_allclose(a, g['actions'][i], rtol=0, atol=1e-7)


def test_oracle_act_ou_matches_reference(golden):
    g = golden('ddpg_ln_act_ou')
    actor = actor_layers(g.sub('model/'))
    x = np.zeros(3)
    for i in range(len(g['obs'])):
        if i == int(g['reset_at']):
            x = np.zeros(3)
        a, x = ddpg_act_ou(g['obs'][i], actor, x, float(g['sigma']), float(g['theta']), float(g['dt']),
                           g['unit_noise'][i])
        np.testing.assert_allclose(a, g['actions'][i], rtol=0, atol=1e-7)
        np.testing.assert_allclose(x, g['ou_states'][i], rtol=0, atol=1e-12)


@pytest.mark.parametrize('tag,kind', [('normal', 'normal'), ('adaptive', 'adaptive_normal')])
def test_oracle_param_noise_matches_reference(golden, tag, kind):
    """Every actor entry of the state dict is perturbed, LayerNorm gains and biases included (param_noise.py:14-23)."""
    g = golden('ddpg_ln_param_noise_' + tag)
    cfg = g.js('cfg')
    actor_keys = [k for k in cfg['keys'] if k.startswith('actor')]
    assert len(actor_keys) == 10 and 'actor.model.seq.5.weight' in actor_keys
    for a in range(cfg['agents']):
        pn = (PN.NormalParameterNoise(cfg['sigma']) if kind == 'normal' else
              PN.AdaptiveNormalParameterNoise(cfg['target_stddev'], cfg['interval'], cfg['alpha'], cfg['sigma']))
        sig_a = float(g['a%d/action_sigma' % a])
        for f in range(cfg['fetches']):
            model = g.sub('f%d/model/' % f)
            draws = iter([g['a%d/f%d/pz/%s' % (a, f, k.replace('.', '/'))] for k in actor_keys])
            pert = pn.apply({k: model[k.replace('.', '/')] for k in actor_keys}, lambda shape: next(draws))
            for k, v in pert.items():
                np.testing.assert_array_equal(v, g['a%d/f%d/pert/%s' % (a, f, k.replace('.', '/'))])
            assert pn.sigma == g['a%d/sigma' % a][f]
            pl = actor_layers({k.replace('.', '/'): v for k, v in pert.items()})
            orig = actor_layers(model)
            for t in range(cfg['acts']):
                x = torch.tensor(g['obs'][f, t]).unsqueeze(0)
                with torch.no_grad():
                    pn.compute_action_distance(R.ddpg_actor(x, orig)[0], R.ddpg_actor(x, pl)[0])
                act = ddpg_act(g['obs'][f, t], pl, sig_a, g['a%d/action_z' % a][f, t])
                np.testing.assert_allclose(act, g['a%d/actions' % a][f, t], rtol=0, atol=2e-6)


@pytest.mark.parametrize('dims', [[9, 20, 12, 3], [64, 300, 200, 8], [17, 45, 33, 1]])
def test_layernorm_image_layout(dims):
    """Gain and bias follow their layer's bias, padded like it; the flat order is the reference's state-dict order."""
    lay, size = R.flat_layout(dims)
    plain, psize = PN.flat_layout(dims)
    assert size == psize + sum(2 * PN._ru(n, 4) for n in dims[1:-1])
    for l, (w, b, K, N, ldw, g, beta) in enumerate(lay):
        assert b == w + K * ldw
        if l + 2 < len(dims):
            assert g == b + ldw and beta == g + ldw
        else:
            assert g is None and beta is None
    stride = R.image_stride(dims)
    pad = R.padding_mask(dims, stride)
    n_params = sum(dims[l] * dims[l + 1] + dims[l + 1] for l in range(len(dims) - 1)) + 2 * sum(dims[1:-1])
    assert int((~pad).sum()) == n_params
    rng = np.random.default_rng(0)
    layers = [tuple(rng.standard_normal(s).astype(np.float32) for s in
                    ([(dims[l + 1], dims[l]), (dims[l + 1],)] + ([(dims[l + 1],)] * 2 if l + 2 < len(dims) else [])))
              for l in range(len(dims) - 1)]
    flat = R.to_flat(layers, dims, stride)
    assert np.all(flat[pad] == 0)
    for e, e2 in zip(layers, R.from_flat(flat, dims)):
        for t, t2 in zip(e, e2):
            np.testing.assert_array_equal(t, t2)

"""DDPG parameter-space noise without a GPU: the oracle (oracle/param_noise.py) against the reference goldens, the
per-actor image layout, the Philox perturbation stream's key, and the agent's reading of param_noise_type."""
import numpy as np
import pytest
import torch

from oracle import nets
from oracle.agent import ddpg_act
from oracle import param_noise as PN
from oracle import philox

KINDS = [('normal', 'normal'), ('adaptive', 'adaptive_normal')]


def _layers(sd, prefix):
    return nets.params_from_state(sd, prefix)


def _dims(cfg):
    return [cfg['D']] + cfg['actor_h'] + [cfg['A']]


def replay_agent(g, a):
    """Replays reference agent `a` of a golden with the oracle and the recorded draws -> (perturbed per fetch,
    actions [F, T, A], sigma per fetch, decisions)."""
    cfg = g.js('cfg')
    if cfg['kind'] == 'normal':
        pn = PN.NormalParameterNoise(cfg['sigma'])
    else:
        pn = PN.AdaptiveNormalParameterNoise(cfg['target_stddev'], cfg['interval'], cfg['alpha'], cfg['sigma'])
    sig_a = float(g['a%d/action_sigma' % a])
    perts, acts, sigmas = [], [], []
    orig = None
    for f in range(cfg['fetches']):
        model = {k: v for k, v in g.sub('f%d/model/' % f).items()}
        draws = iter([g['a%d/f%d/pz/%s' % (a, f, k.replace('.', '/'))] for k in cfg['keys'] if k.startswith('actor')])
        params = {k: model[k.replace('.', '/')] for k in cfg['keys'] if k.startswith('actor')}
        orig = _layers(model, 'actor/model/')
        pert = pn.apply(params, lambda shape: next(draws))
        perts.append(pert)
        sigmas.append(pn.sigma)
        pl = _layers({k.replace('.', '/'): v for k, v in pert.items()}, 'actor/model/')
        out = []
        for t in range(cfg['acts']):
            x = torch.tensor(g['obs'][f, t]).unsqueeze(0)
            with torch.no_grad():
                pi = nets.ddpg_actor(x, pl)[0]
                pn.compute_action_distance(nets.ddpg_actor(x, orig)[0], pi)
            out.append(ddpg_act(g['obs'][f, t], pl, sig_a, g['a%d/action_z' % a][f, t]))
        acts.append(np.stack(out))
    return perts, np.stack(acts), sigmas, getattr(pn, 'decisions', [])


@pytest.mark.parametrize('tag,kind', KINDS)
def test_oracle_reproduces_reference(golden, tag, kind):
    g = golden('ddpg_param_noise_' + tag)
    cfg = g.js('cfg')
    assert cfg['kind'] == kind
    for a in range(cfg['agents']):
        perts, acts, sigmas, decisions = replay_agent(g, a)
        for f in range(cfg['fetches']):
            for k, v in perts[f].items():
                np.testing.assert_array_equal(v, g['a%d/f%d/pert/%s' % (a, f, k.replace('.', '/'))])
        assert sigmas == list(g['a%d/sigma' % a])                 # float64, exact
        np.testing.assert_allclose(acts, g['a%d/actions' % a], rtol=0, atol=2e-6)
        if kind == 'adaptive_normal':
            assert len(decisions) == cfg['fetches'] - 1            # the first apply comes before any act
            exp = ['down' if s1 < s0 else 'up' for s0, s1 in zip(g['a%d/sigma' % a][:-1], g['a%d/sigma' % a][1:])]
            assert decisions == exp


def test_adaptive_golden_covers_both_decisions(golden):
    g = golden('ddpg_param_noise_adaptive')
    steps = set()
    for a in range(3):
        s = g['a%d/sigma' % a]
        steps |= {'down' if s1 < s0 else 'up' for s0, s1 in zip(s[:-1], s[1:])}
    assert steps == {'up', 'down'}


def test_mean_is_latest_distance_over_acts_since_apply():
    """The dist / i quirk: the distance is overwritten at i = 0, 10, 20 and divided by all 23 acts."""
    pn = PN.AdaptiveNormalParameterNoise(target_stddev=1.0, compute_dist_interval=10, alpha=2.0, sigma=1.0)
    for i in range(23):
        pn.compute_action_distance(np.zeros(2, np.float32), np.full(2, float(i), np.float32))
    assert float(pn.total_action_distance) == pytest.approx(20 * np.sqrt(2), rel=1e-6)
    mean = pn.total_action_distance / pn.i
    assert mean.dtype == torch.float32 and float(mean) == pytest.approx(20 * np.sqrt(2) / 23, rel=1e-6)
    pn.apply({}, None)
    assert pn.sigma == 0.5 and pn.i == 0


@pytest.mark.parametrize('dims', [[64, 300, 200, 8], [17, 48, 32, 3], [5, 7, 1], [9, 20, 12, 3]])
def test_image_layout(dims):
    lay, size = PN.flat_layout(dims)
    stride = PN.image_stride(dims)
    assert stride % 32 == 0 and size <= stride < size + 32
    n_params = sum(dims[l] * dims[l + 1] + dims[l + 1] for l in range(len(dims) - 1))
    pad = PN.padding_mask(dims, stride)
    assert int((~pad).sum()) == n_params
    rng = np.random.default_rng(0)
    layers = [(rng.standard_normal((dims[l + 1], dims[l])).astype(np.float32),
               rng.standard_normal(dims[l + 1]).astype(np.float32)) for l in range(len(dims) - 1)]
    flat = PN.to_flat(layers, dims, stride)
    assert np.all(flat[pad] == 0)
    for (w, b), (w2, b2) in zip(layers, PN.from_flat(flat, dims)):
        np.testing.assert_array_equal(w, w2)
        np.testing.assert_array_equal(b, b2)
    if dims == [64, 300, 200, 8]:
        assert n_params == 81308 and stride == 81312


def test_image_stride_matches_agent():
    from surreal_b200.agent.ddpg_agent import param_noise_stride
    for dims in ([64, 300, 200, 8], [17, 48, 32, 3], [5, 7, 1]):
        assert param_noise_stride(PN.flat_layout(dims)[1]) == PN.image_stride(dims)


def test_perturbation_stream_is_its_own():
    """The perturbation draws differ per actor and per fetch and do not reuse the action-noise key."""
    z00 = PN.param_noise_unit(5, 0, 0, 64)
    z01 = PN.param_noise_unit(5, 0, 1, 64)
    z10 = PN.param_noise_unit(5, 1, 0, 64)
    assert not np.array_equal(z00, z01) and not np.array_equal(z00, z10)
    x, y, _, _ = philox.philox4x32_10(np.uint64(5), np.uint64(0), np.uint64(0))
    a, _ = PN.box_muller_f64(x, y)
    assert float(a) != z00[0]
    big = PN.param_noise_unit(5, 3, 2, 200000)
    assert abs(big.mean()) < 0.01 and abs(big.std() - 1.0) < 0.01


def test_perturb_rounds_once():
    w = np.array([1.0, -2.5, 3e-8], dtype=np.float32)
    z = np.array([0.3, 1e-9, -0.7])
    got = PN.perturb({'w': w}, 0.05, lambda shape: z)['w']
    np.testing.assert_array_equal(got, (w.astype(np.float64) + 0.05 * z).astype(np.float32))


@pytest.mark.parametrize('value,expected', [(None, None), ('normal', 'normal'), ('adaptive_normal', 'adaptive_normal'),
                                            ('gaussian', None)])
def test_param_noise_type_config(monkeypatch, value, expected):
    """The agent reads param_noise_type as the reference does (ddpg_agent.py:120-147); unknown values mean none.  The
    agent itself needs a GPU, so its constructor is stopped right after the decision."""
    from surreal_b200.agent import ddpg_agent as M
    from helpers import ddpg_configs
    lc, ec, sc = ddpg_configs()
    lc.algo.exploration.param_noise_type = value
    seen = {}

    class Stop(Exception):
        pass

    def model(*a, **k):
        raise Stop

    monkeypatch.setattr(M.torch.cuda, 'is_available', lambda: True)
    monkeypatch.setattr(M.torch.cuda, 'current_device', lambda: 0)
    monkeypatch.setattr(M, 'DDPGModel', model)
    for mode, exp in (('training', expected), ('eval_stochastic', expected), ('eval_deterministic', None)):
        ag = M.DDPGAgent.__new__(M.DDPGAgent)
        with pytest.raises(Stop):
            M.DDPGAgent.__init__(ag, lc, ec, sc, 0, mode)
        seen[mode] = ag.param_noise_type
        assert ag.param_noise_type == exp, (mode, value)

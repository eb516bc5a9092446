"""Stacked LSTM stems (algo.rnn.rnn_layer > 1) on the CPU: the oracle learner and agent against goldens the REAL reference
produced at rnn_layer = 2 and 3 (tests/golden/make_golden_rnn_layers.py), the float64 stacked LSTM of
grad_ref_stacked against torch.nn.LSTM(num_layers = L), and the record layout of the cells (utils.rnn_cell_layout)."""
import numpy as np
import pytest
import torch

from oracle.agent import ppo_act_rnn
from oracle.ppo_rnn import OraclePPOLearnerRNN
from test_oracle_golden import _ppo_model, _state_matches

T = torch.tensor


@pytest.mark.parametrize('tag', ['rnn2_clip', 'rnn2_adapt', 'rnn3_clip'])
def test_oracle_learner_stacked_lstm(golden, tag):
    """learn() + publish of the RNN oracle with L layers against the reference: onetime_infos [B, L, H], every layer of
    the stem trained by both optimisers.  Same bars as the one-layer goldens (test_oracle_golden.py)."""
    torch.set_num_threads(1)
    g = golden('ppo_learn_' + tag)
    cfg, hyper, stats = g.js('cfg'), g.js('hyper'), g.js('stats')
    Lr = cfg['rnn_layer']
    assert Lr == int(tag[3])
    init = g.sub('init/')
    actor, log_var, critic, zf = _ppo_model(init)
    lstm = {k.split('/', 1)[1]: init[k] for k in init.keys() if k.startswith('rnn_stem/')}
    assert sorted(lstm) == sorted('%s_%s_l%d' % (a, b, k) for a in ('weight', 'bias') for b in ('ih', 'hh') for k in range(Lr))
    assert lstm['weight_ih_l1'].shape == (4 * cfg['rnn_hidden'], cfg['rnn_hidden'])
    L = OraclePPOLearnerRNN(actor, log_var, critic, zf, lstm, cfg['A'], cfg['n_step'], cfg['B'], cfg['horizon'],
                            cfg['rnn_hidden'], Lr, ppo_mode=cfg['mode'], lr_actor=cfg['lr'],
                            lr_critic=cfg['lr'], exp_interval=cfg['exp_interval'])
    for it in range(cfg['iters']):
        b = g.sub('it%d/' % it)
        assert b['h0'].shape == (cfg['B'], Lr, cfg['rnn_hidden'])
        st = L.learn(dict(obs=b['obs'], obs_next=b['obs_next'], actions=b['actions'], rewards=b['rewards'],
                          dones=b['dones'], pd=b['pd'], h0=b['h0'], c0=b['c0']))
        np.testing.assert_allclose(L.last_adv.numpy(), b['adv'], rtol=0, atol=1e-6)
        np.testing.assert_allclose(L.last_ret.numpy(), b['ret'], rtol=0, atol=1e-6)
        L.publish_parameter()
        assert L.n_policy_epochs[-1] == hyper[it]['n_policy_epochs']
        for k, v in stats[it].items():
            assert st[k] == pytest.approx(v, rel=1e-5, abs=1e-6), k
        after = g.sub('it%d/after/' % it)
        _state_matches(L, after, atol=1e-6)
        for name, p in L.rnn.named_parameters():
            np.testing.assert_allclose(p.detach().numpy(), after['rnn_stem/' + name], rtol=0, atol=1e-6, err_msg=name)
        for name, p in L.ref_rnn.named_parameters():
            np.testing.assert_allclose(p.detach().numpy(), b['ref/rnn_stem/' + name], rtol=0, atol=1e-6, err_msg=name)
        if cfg['mode'] == 'clip':
            assert L.clip_epsilon == pytest.approx(hyper[it]['clip_epsilon'], rel=1e-12)
        else:
            assert L.beta == pytest.approx(hyper[it]['beta'], rel=1e-12)
        assert L.exp_counter == hyper[it]['exp_counter']
    if tag == 'rnn2_adapt':                               # the fixture exercises the KL early stop
        assert all(h['n_policy_epochs'] < cfg['epoch_policy'] for h in hyper)


def test_oracle_agent_stacked_lstm(golden):
    """The actor side at rnn_layer = 2: cells (2, 1, H) carried between steps, onetime_infos (2, H) per step, reset()."""
    torch.set_num_threads(1)
    g = golden('ppo_act_rnn2')
    sd = g.sub('model/')
    actor, log_var, _, zf = _ppo_model(sd)
    Hd = int(g['rnn_hidden'])
    assert g['h_before'].shape == (len(g['obs']), 2, Hd)
    lstm = torch.nn.LSTM(11, Hd, 2, batch_first=True)
    lstm.load_state_dict({k.split('/', 1)[1]: T(sd[k]) for k in sd.keys() if k.startswith('rnn_stem/')})
    zero = lambda: (torch.zeros(2, 1, Hd), torch.zeros(2, 1, Hd))   # noqa: E731
    cells = zero()
    for i in range(len(g['obs'])):
        if i == int(g['reset_at']):
            cells = zero()
        a, pdv, onetime, cells = ppo_act_rnn(g['obs'][i], actor, log_var, zf, lstm, cells, float(g['noise']), eps=g['eps'][i])
        np.testing.assert_allclose(onetime[0], g['h_before'][i], rtol=0, atol=1e-7)
        np.testing.assert_allclose(onetime[1], g['c_before'][i], rtol=0, atol=1e-7)
        np.testing.assert_allclose(pdv, g['pds'][i], rtol=0, atol=1e-7)
        np.testing.assert_allclose(a, g['actions'][i], rtol=0, atol=1e-7)
    hb = g['h_before']
    assert np.abs(hb[1, 1]).max() > 0 and np.abs(hb[int(g['reset_at'])]).max() == 0
    assert np.abs(hb[2, 0] - hb[2, 1]).max() > 1e-3                  # the two layers carry different cells


@pytest.mark.parametrize('B,L,D,H,layers', [(3, 5, 7, 6, 2), (2, 9, 4, 11, 3), (1, 1, 3, 1, 2)])
def test_lstm_stack_matches_torch_float64(B, L, D, H, layers):
    """lstm_stack against torch.nn.LSTM(num_layers = layers) in float64: outputs, last cells of every layer, and the
    gradients of every layer's weights."""
    from grad_ref_stacked import lstm_stack
    torch.manual_seed(B * 100 + L * 10 + layers)
    ref = torch.nn.LSTM(D, H, layers, batch_first=True).double()
    x = torch.randn(B, L, D, dtype=torch.float64)
    h0, c0 = torch.randn(layers, B, H, dtype=torch.float64) * 0.5, torch.randn(layers, B, H, dtype=torch.float64) * 0.5
    out, (hn, cn) = ref(x, (h0, c0))
    seed = torch.randn(B, L, H, dtype=torch.float64)
    names = ['%s_%s_l%d' % (a, b, k) for k in range(layers) for a, b in (('weight', 'ih'), ('weight', 'hh'), ('bias', 'ih'), ('bias', 'hh'))]
    g_ref = torch.autograd.grad((out * seed).sum(), [getattr(ref, n) for n in names])
    W = [getattr(ref, n).detach().clone().requires_grad_(True) for n in names]
    rs = lstm_stack(x, list(h0), list(c0), [W[4 * k:4 * k + 4] for k in range(layers)])
    assert torch.allclose(rs[-1]['h'], out, rtol=0, atol=1e-12)
    for k in range(layers):
        assert torch.allclose(rs[k]['h_last'], hn[k], rtol=0, atol=1e-12)
        assert torch.allclose(rs[k]['c_last'], cn[k], rtol=0, atol=1e-12)
    g = torch.autograd.grad((rs[-1]['h'] * seed).sum(), W)
    for n, a, b in zip(names, g, g_ref):
        assert torch.allclose(a, b, rtol=0, atol=1e-11), n


def _cfgs(layers, H=10, D=11, rnn=True):
    from helpers import ppo_configs
    lc, ec, sc = ppo_configs(D=D)
    lc.algo.rnn.if_rnn_policy = rnn
    lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = H, layers
    return lc, ec, sc


@pytest.mark.parametrize('layers', [1, 2, 3])
def test_cell_layout(layers):
    """The one owner of the cells' columns: [obs | h_0 .. h_{L-1} | c_0 .. c_{L-1}], i.e. onetime_infos [L, H] flattened
    layer-major; record_obs_dim is its width.  At one layer: [obs | h | c]."""
    from surreal_b200 import utils as U
    D, H = 11, 10
    lc, ec, _ = _cfgs(layers, H, D)
    cl = U.rnn_cell_layout(lc, ec)
    assert (cl.layers, cl.hidden, cl.obs_dim) == (layers, H, D)
    assert (cl.h_col, cl.c_col, cl.width) == (D, D + layers * H, D + 2 * layers * H)
    assert U.record_obs_dim(lc, ec) == cl.width
    rng = np.random.default_rng(layers)
    B = 4
    h, c = rng.standard_normal((B, layers, H)), rng.standard_normal((B, layers, H))
    rows = np.full((B, 6, cl.width), np.nan)
    cl.h(rows[:, 0])[...] = h.reshape(B, -1)
    cl.c(rows[:, 0])[...] = c.reshape(B, -1)
    assert np.isnan(rows[:, 0, :D]).all() and np.isnan(rows[:, 1:]).all()
    np.testing.assert_array_equal(cl.h(rows[:, 0]).reshape(B, layers, H), h)                # [B, L, H] round trip
    np.testing.assert_array_equal(cl.c(rows[:, 0]).reshape(B, layers, H), c)
    for k in range(layers):
        np.testing.assert_array_equal(cl.h(rows[:, 0], k), h[:, k])
        np.testing.assert_array_equal(cl.c(rows[:, 0], k), c[:, k])
    if layers == 1:
        np.testing.assert_array_equal(rows[:, 0, D:D + H], h[:, 0])
        np.testing.assert_array_equal(rows[:, 0, D + H:], c[:, 0])
    t = torch.tensor(rows)
    assert tuple(cl.h(t[:, 0]).unflatten(1, (layers, H)).shape) == (B, layers, H)        # the replay's [B, L, H] views


def test_cell_layout_feed_forward_and_bad_depth():
    from surreal_b200 import utils as U
    from surreal_b200.session import ConfigError
    lc, ec, _ = _cfgs(2, rnn=False)
    assert U.rnn_cell_layout(lc, ec) is None and U.record_obs_dim(lc, ec) == 11
    for bad in (0, -1):
        lc, ec, _ = _cfgs(bad)
        with pytest.raises(ConfigError):
            U.rnn_cell_layout(lc, ec)
        with pytest.raises(ConfigError):
            U.record_obs_dim(lc, ec)
    lc, ec, _ = _cfgs(1)
    assert U.record_obs_dim(lc, ec) == 11 + 20

"""RNN mode on the GPU (SURVEY §8f rank 2; the reference's DEFAULT PPO config): LSTM stem kernels vs torch.nn.LSTM and,
over their whole shape envelope, vs a float64 cell loop (tests/grad_ref.py lstm); the learner's row gather / z-filter;
PPOAgent.act at up to 1024 actors vs float64 steps; the
RNN-mode PPOLearner against goldens produced by the REFERENCE's PPOLearner (LSTM trained by both optimisers, horizon GAE
over eff_len positions, initial cells from onetime_infos; ppo.py:389-406,507-525), PPOAgent.act with cell hand-off against
the reference golden, and the whole default config end to end (actors -> HBM staging with the cells riding in the
observation rows -> FIFO -> learner)."""
import copy

import numpy as np
import pytest
import torch

from helpers import ppo_configs, ref_state_dict

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
LOSS_STATS = ['_surr_loss', '_clip_surr_loss', '_kl_loss_adapt', '_entropy', '_pol_kl', '_val_loss', '_avg_return_targ',
              '_avg_log_sig', '_avg_behave_likelihood', '_avg_is_weight', '_ref_behave_diff', 'obs_running_mean',
              'obs_running_square', 'obs_running_std']


@pytest.mark.parametrize('B,L,D,H', [(8, 16, 17, 100), (5, 7, 11, 10), (64, 26, 17, 100)])
def test_lstm_forward_backward_match_torch(B, L, D, H):
    from surreal_b200.model.lstm_stem import LSTMStem, RnnTrainer
    g = torch.Generator().manual_seed(B + L + H)
    ref = torch.nn.LSTM(D, H, 1, batch_first=True)
    stem = LSTMStem(D, H, DEV)
    stem.load_torch({k: v.detach() for k, v in ref.state_dict().items()})
    x = torch.randn(B, L, D, generator=g)
    h0, c0 = torch.randn(1, B, H, generator=g) * 0.5, torch.randn(1, B, H, generator=g) * 0.5
    out, (hn, cn) = ref(x, (h0, c0))
    dout = torch.randn(B, L, H, generator=g)
    out.backward(dout)
    tr = RnnTrainer(stem, B, L)
    xf = torch.zeros(B * L, (D + 3) // 4 * 4, device=DEV)[:, :D]
    xf.copy_(x.reshape(B * L, D))
    h0d, c0d = h0[0].to(DEV).contiguous(), c0[0].to(DEV).contiguous()
    h = tr.forward(xf, h0d, c0d, H)
    torch.cuda.synchronize()
    assert float((h.cpu().reshape(B, L, H) - out.detach()).abs().max()) <= 1e-5
    dh = torch.zeros(B * L, (H + 3) // 4 * 4, device=DEV)
    dh[:, :H].copy_(dout.reshape(B * L, H))
    tr.backward(dh)
    torch.cuda.synchronize()
    gsum = tr.slabs.sum(0)
    wi, bi = stem.ih.get_layer(0, gsum[:stem.ih.size])
    wh, bh = stem.hh.get_layer(0, gsum[stem.ih.size:])
    scale = max(1.0, float(ref.weight_hh_l0.grad.abs().max()))
    assert float((wi.cpu() - ref.weight_ih_l0.grad).abs().max()) <= 2e-5 * scale
    assert float((wh.cpu() - ref.weight_hh_l0.grad).abs().max()) <= 2e-5 * scale
    assert float((bi.cpu() - ref.bias_ih_l0.grad).abs().max()) <= 2e-5 * scale
    assert float((bh.cpu() - ref.bias_hh_l0.grad).abs().max()) <= 2e-5 * scale


NAN = float('nan')
# (B, L, D, H, cells, splits).  cells: 'given' = contiguous [B, H] initial cells (then also run in place, h_last = h0,
# c_last = c0, as the agent does), 'none' = h0 = c0 = None (zeros), 'wide' = cells inside wider rows, as the learner
# reads them out of its observation records (ld_cells = (n+1)(D+2H), every other element NaN).
LSTM_CASES = [(1, 1, 1, 1, 'given', 1), (3, 2, 5, 7, 'none', 2), (6, 26, 3, 31, 'wide', 1), (64, 26, 17, 100, 'wide', 16),
              (5, 129, 9, 100, 'given', 3), (4096, 2, 33, 255, 'wide', 16), (16, 130, 64, 256, 'given', 7),
              (1024, 1, 17, 256, 'none', 8), (2, 26, 17, 256, 'given', 16)]
# Bars per output; the worst error measured on an H100 80GB HBM3 over LSTM_CASES is in the comment.  The forward
# outputs are O(1) and are held to max |err|.  dpre and the weight gradients are held to relative L2 and to
# max |err| / max |g64|.  The worst cases are the longest sequences and H = 255 / 256.
LSTM_BAR = {'h': 2e-6,          # 2.6e-7 (h_out, h_prev, h_last)
            'gates': 5e-6,      # 7.6e-7
            'c': 5e-6,          # 5.5e-7 (c_seq, c_last)
            'dpre': 4e-6,       # 4.3e-7
            'dW': 5e-6}         # 6.3e-7 (dW_ih, dW_hh, db_ih, db_hh over 1..16 slabs)


def _cells_buffers(case_cells, B, H, D, gen):
    """-> (h0, c0, ld_cells, h64, c64): the initial cells as the kernel reads them and as float64 [B, H] (or None)."""
    if case_cells == 'none':
        return None, None, 0, None, None
    h = torch.randn(B, H, generator=gen, device=DEV) * 0.5
    c = torch.randn(B, H, generator=gen, device=DEV) * 0.8
    if case_cells == 'given':
        return h.clone(), c.clone(), H, h.double(), c.double()
    n1 = 26                                                                         # rows of n_step + 1 = 26 observations
    rows = torch.full((B, n1, D + 2 * H), NAN, device=DEV)
    rows[:, 0, D:D + H], rows[:, 0, D + H:] = h, c
    return rows[:, 0, D:D + H], rows[:, 0, D + H:], rows.stride(0), h.double(), c.double()


def _err(got, exp):
    e = (got.double() - exp).abs()
    return float(e.max()), float((got.double() - exp).norm()) / max(float(exp.norm()), 1e-30), \
        float(e.max()) / max(float(exp.abs().max()), 1e-30)


@pytest.mark.parametrize('B,L,D,H,cells,splits', LSTM_CASES)
def test_lstm_kernels_match_float64(B, L, D, H, cells, splits):
    """sb200_lstm_forward_f32 / sb200_lstm_backward_f32 through LSTMStem / RnnTrainer against grad_ref.lstm in float64:
    every saved output (h_out, h_prev, gates, c_seq, h_last, c_last), the gate pre-activation gradient dpre itself and
    the four weight gradients after the slab reduction.  NaN sentinels sit in the padding columns of h_out / h_prev
    (which must stay untouched) and in the columns of dh_out at or past H (which must not be read)."""
    import grad_ref as R
    from surreal_b200.model.lstm_stem import LSTMStem, RnnTrainer
    gen = torch.Generator(device=DEV).manual_seed(B * 7 + L * 3 + H)
    k = 1.0 / H ** 0.5
    u = lambda *s: (torch.rand(*s, generator=gen, device=DEV) * 2 - 1) * k  # noqa: E731
    w = {'weight_ih_l0': u(4 * H, D), 'weight_hh_l0': u(4 * H, H), 'bias_ih_l0': u(4 * H), 'bias_hh_l0': u(4 * H)}
    stem = LSTMStem(D, H, DEV)
    stem.load_torch(w)
    h0, c0, ld, h64, c64 = _cells_buffers(cells, B, H, D, gen)
    Rn, Hp = B * L, (H + 3) // 4 * 4
    x = torch.randn(B, L, D, generator=gen, device=DEV)
    xf = torch.zeros(Rn, (D + 3) // 4 * 4, device=DEV)[:, :D]
    xf.copy_(x.reshape(Rn, D))
    tr = RnnTrainer(stem, B, L, splits=splits)
    for name in ('h_out', 'h_prev'):
        tr.bufs[name] = torch.full((Rn, Hp), NAN, device=DEV)[:, :H]
    h_out = tr.forward(xf, h0, c0, ld)
    dout = torch.randn(B, L, H, generator=gen, device=DEV)
    dh = torch.full((Rn, Hp + 4), NAN, device=DEV)
    dh[:, :H] = dout.reshape(Rn, H)
    tr.backward(dh)
    torch.cuda.synchronize()
    # float64 reference: the same fp32 inputs and weights
    W = [R.f64(w[k_]).requires_grad_(True) for k_ in ('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0')]
    r = R.lstm(R.f64(x), h64, c64, *W)
    seed = R.f64(dout)
    gs = torch.autograd.grad((r['h'] * seed).sum(), W + r['pre'])
    h_ref = r['h'].detach().reshape(Rn, H)
    hp_ref = torch.cat([(h64 if h64 is not None else torch.zeros(B, H, dtype=torch.float64, device=DEV))[:, None],
                        r['h'].detach()[:, :-1]], 1).reshape(Rn, H)
    worst = {}

    def fwd(name, got, exp):
        e = _err(got, exp)[0]
        worst[name] = max(worst.get(name, 0.0), e)
        assert e <= LSTM_BAR[name], (name, e)

    base = h_out._base if h_out._base is not None else h_out
    assert bool(torch.isnan(base[:, H:]).all()), 'h_out padding columns written'
    assert bool(torch.isnan(tr.bufs['h_prev']._base[:, H:]).all()), 'h_prev padding columns written'
    fwd('h', h_out, h_ref)
    fwd('h', tr.bufs['h_prev'], hp_ref)
    fwd('gates', tr.bufs['gates'], r['gates'].detach().reshape(Rn, 4 * H))
    fwd('c', tr.bufs['c_seq'], r['c'].detach().reshape(Rn, H))
    dpre_ref = torch.stack(gs[4:], 1).reshape(Rn, 4 * H)
    _, rel, mx = _err(tr.dpre, dpre_ref)
    worst['dpre'] = max(rel, mx)
    assert rel <= LSTM_BAR['dpre'] and mx <= LSTM_BAR['dpre'], ('dpre', rel, mx)
    g = tr.slabs.double().sum(0).float()
    wi, bi = stem.ih.get_layer(0, g[:stem.ih.size])
    wh, bh = stem.hh.get_layer(0, g[stem.ih.size:])
    for got, exp, nm in ((wi, gs[0], 'dW_ih'), (wh, gs[1], 'dW_hh'), (bi, gs[2], 'db_ih'), (bh, gs[3], 'db_hh')):
        _, rel, mx = _err(got, exp)
        worst['dW'] = max(worst.get('dW', 0.0), rel, mx)
        assert rel <= LSTM_BAR['dW'] and mx <= LSTM_BAR['dW'], (nm, rel, mx)
    # the final cells, written to their own buffers and, as the agent does, in place over the initial cells
    bufs = stem.buffers(B, L, save=False)
    hl, cl = torch.full((B, H), NAN, device=DEV), torch.full((B, H), NAN, device=DEV)
    stem.forward(xf, h0, c0, ld, B, L, bufs, h_last=hl, c_last=cl)
    torch.cuda.synchronize()
    assert torch.equal(bufs['h_out'], h_out), 'h_out depends on whether h_last / c_last are written'
    fwd('h', hl, r['h_last'].detach())
    fwd('c', cl, r['c_last'].detach())
    if cells == 'given':
        stem.forward(xf, h0, c0, ld, B, L, bufs, h_last=h0, c_last=c0)
        torch.cuda.synchronize()
        assert torch.equal(h0, hl) and torch.equal(c0, cl), 'in-place h_last = h0 / c_last = c0 differs'
    print('measured lstm', B, L, D, H, cells, worst)


@pytest.mark.parametrize('B,n,E,D,H', [(64, 25, 16, 17, 100), (3, 1, 1, 5, 7), (1024, 25, 1, 64, 256)])
def test_rows_zfilter_learner_strides(B, n, E, D, H):
    """sb200_rows_zfilter_f32 as the learner calls it: rows b*(n+1) + t of the observation records (D features, then
    the 2H cells), all n+1 steps and the eff_len prefix, with the z-filter (columns at the eps floor of std, values past
    the +-5 clamp) and as a plain gather (zf = None).  Against grad_ref.zfilter: measured worst 2.2e-7 (bar
    1e-6 (1 + |z|) elementwise); the gather is exact."""
    import grad_ref as R
    from surreal_b200.model.lstm_stem import rows_zfilter
    gen = torch.Generator(device=DEV).manual_seed(B + n + D)
    Dp = D + 2 * H
    cnt = 300.0
    mean = torch.randn(D, generator=gen, device=DEV)
    var = 0.3 + torch.rand(D, generator=gen, device=DEV)
    mean[0], var[0] = 0.5, 0.0                                         # exactly representable: std = 0, floored at eps
    zs = torch.cat([mean * cnt, (var + mean ** 2) * cnt, torch.tensor([cnt], device=DEV)])
    obs = torch.full((B, n + 1, Dp), NAN, device=DEV)
    obs[:, :, :D] = mean + torch.randn(B, n + 1, D, generator=gen, device=DEV) * var.sqrt()
    obs[:, :, 0] = 0.5 + 1e-6 * torch.randint(-8, 9, (B, n + 1), generator=gen, device=DEV)   # (x - 0.5) / eps in [-0.8, 0.8]
    obs[:, ::3, D - 1] += 20.0 * var[D - 1].sqrt()                     # past the +5 clamp
    obs[:, 1::3, D - 1] -= 20.0 * var[D - 1].sqrt()
    for L in sorted({n + 1, E}):
        for stats in (zs, None):
            out = torch.full((B * L, (D + 3) // 4 * 4 + 4), NAN, device=DEV)
            rows_zfilter(obs, Dp, (n + 1) * Dp, B, L, D, stats, 1e-5, out)
            torch.cuda.synchronize()
            x = obs[:, :L, :D].reshape(B * L, D)
            assert bool(torch.isnan(out[:, D:]).all()), 'columns past D written'
            if stats is None:
                assert torch.equal(out[:, :D], x)
                continue
            z = R.zfilter(x, zs)
            if L == n + 1:
                assert float(z.abs().max()) == 5.0 and float(z[:, 0].abs().max()) > 0.1
            err = float(((out[:, :D].double() - z).abs() / (1 + z.abs())).max())
            print('measured zfilter', B, L, D, err)
            assert err <= 1e-6, err


def _rnn_cfg(cfg, B=None):
    lc, ec, sc = ppo_configs(D=cfg['D'], A=cfg['A'], actor_h=cfg['actor_h'], critic_h=cfg['critic_h'], n_step=cfg['n_step'],
                             stride=cfg['n_step'], B=B or cfg['B'], mode=cfg['mode'], lr=cfg['lr'], exp_interval=cfg['exp_interval'])
    lc.algo.rnn.if_rnn_policy = True
    lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = cfg['horizon'], cfg['rnn_hidden'], cfg['rnn_layer']
    return lc, ec, sc


@pytest.mark.parametrize('tag', ['rnn_clip', 'rnn_adapt', 'rnn_adapt_biglr'])
def test_ppo_learn_rnn_matches_reference(golden, tag):
    from surreal_b200.learner import PPOLearner
    g = golden('ppo_learn_' + tag)
    cfg, hyper, stats = g.js('cfg'), g.js('hyper'), g.js('stats')
    lc, ec, sc = _rnn_cfg(cfg)
    L = PPOLearner(lc, ec, sc)
    L.model.load_state_dict(ref_state_dict(g.sub('init/')))
    L.ref_target_model.update_target_params(L.model)
    lr, E = cfg['lr'], cfg['n_step'] - cfg['horizon'] + 1
    for it in range(cfg['iters']):
        b = g.sub('it%d/' % it)
        st = L.learn({'obs': {'low_dim': {'flat_inputs': b['obs']}}, 'obs_next': {'low_dim': {'flat_inputs': b['obs_next']}},
                      'actions': b['actions'], 'rewards': b['rewards'], 'dones': b['dones'], 'persistent_infos': [b['pd']],
                      'onetime_infos': [b['h0'], b['c0']]})
        L.publish_parameter(it, message='')
        torch.cuda.synchronize()
        assert L._adv.shape == (cfg['B'], E)
        assert float((L._adv.cpu() - torch.tensor(b['adv'])).abs().max()) <= 1e-5
        rms = float(np.sqrt((b['ret'] ** 2).mean()))
        assert float((L._ret.cpu() - torch.tensor(b['ret'])).abs().max()) <= 1e-5 * max(1.0, rms)
        assert L.last_n_policy_epochs == hyper[it]['n_policy_epochs'], 'KL early stop diverged'
        for k, v in stats[it].items():
            assert k in st, k
            tol = 1e-5 * max(1.0, abs(v)) if k in LOSS_STATS else 2e-4 * max(1.0, abs(v))
            if k == '_val_explained_var':
                tol = 1e-4
            assert abs(st[k] - v) <= tol, '%s it%d: got %.9g expected %.9g' % (k, it, st[k], v)
        after = ref_state_dict(g.sub('it%d/after/' % it))
        got = L.model.state_dict()
        assert set(after) <= set(got), sorted(set(after) - set(got))
        worst = 0.0
        for k, e in after.items():
            gk = got[k].cpu().reshape(e.shape)
            if k.startswith('z_filter'):     # running sums of +-O(1) values: fp32 summation order, relative to the vector's scale
                assert float((gk - e).abs().max()) <= 1e-6 * max(1.0, float(e.abs().max())), k
                continue
            worst = max(worst, float((gk - e).abs().max()))
        assert worst <= max(2e-6, 0.02 * lr), 'params drifted by %.3e' % worst
        if cfg['mode'] == 'clip':
            assert L.clip_epsilon == pytest.approx(hyper[it]['clip_epsilon'], rel=1e-12)
        else:
            assert L.beta == pytest.approx(hyper[it]['beta'], rel=1e-12)
        assert L.exp_counter == hyper[it]['exp_counter']


def test_ppo_agent_act_rnn_matches_reference(golden):
    """One actor, seven steps: cells carried between steps, the PRE-step cells are the onetime_info, reset() zeroes them."""
    from surreal_b200.agent import PPOAgent
    g = golden('ppo_act_rnn')
    Hd = int(g['rnn_hidden'])
    cfg = dict(D=11, A=3, actor_h=[32, 24], critic_h=[28, 20], n_step=4, B=4, mode='clip', lr=1e-4, exp_interval=64, horizon=2,
               rnn_hidden=Hd, rnn_layer=1)
    lc, ec, sc = _rnn_cfg(cfg)
    ec.num_envs = 1
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    ag.model.load_state_dict(ref_state_dict(g.sub('model/')))
    ag.set_noise(np.array([float(g['noise'])]))
    for i in range(len(g['obs'])):
        if i == int(g['reset_at']):
            ag.reset()
        a, info = ag.act(g['obs'][i], eps=g['eps'][i])
        np.testing.assert_allclose(info[0][0], g['h_before'][i], rtol=0, atol=2e-6)
        np.testing.assert_allclose(info[0][1], g['c_before'][i], rtol=0, atol=2e-6)
        np.testing.assert_allclose(info[1][0], g['pds'][i], rtol=0, atol=2e-6)
        np.testing.assert_allclose(a, g['actions'][i], rtol=0, atol=5e-6)


@pytest.mark.parametrize('D', [5, 40])
def test_ppo_model_forward_refuses_rnn(D):
    """PPOModel.forward_actor / forward_critic have no cells to run an LSTM stem from: an RNN model raises instead of
    applying the heads to raw observations, whether the observation is narrower than rnn_hidden (16) or not."""
    from surreal_b200.model.ppo_net import PPOModel
    cfg = dict(D=D, A=3, actor_h=[32, 24], critic_h=[28, 20], n_step=4, B=4, mode='clip', lr=1e-4, exp_interval=64, horizon=2,
               rnn_hidden=16, rnn_layer=1)
    lc, ec, sc = _rnn_cfg(cfg)
    m = PPOModel(ec.obs_spec, 3, lc.model, use_z_filter=lc.algo.use_z_filter, rnn_config=lc.algo.rnn, device=DEV)
    obs = torch.randn(8, D, device=DEV)
    with pytest.raises(NotImplementedError):
        m.forward_actor(obs)
    with pytest.raises(NotImplementedError):
        m.forward_critic(obs)


ACT_BAR = 2e-6        # one step from the agent's own cells: pd, action and the new cells, max |err|; measured 2.6e-7
DRIFT_BAR = 1.5e-6    # free-running float64 trajectory against the agent's cells over 40 steps, max |err|; measured 1.6e-7


@pytest.mark.parametrize('N,H', [(1, 100), (64, 256), (1024, 100), (1024, 256)])
def test_ppo_agent_act_rnn_at_scale(N, H):
    """PPOAgent in RNN mode for 40 steps with injected eps, per-actor noise and a reset() at step 23.  Every step: the
    onetime cells are exactly the cells held before the step (zeros right after the reset), and pd, the action and the
    cells written in place (h_last = h0, c_last = c0) match one float64 step taken from those cells.  The free-running
    float64 trajectory stays within DRIFT_BAR of the agent's cells."""
    import grad_ref as R
    from surreal_b200.agent import PPOAgent
    D, A, steps, reset_at = 17, 6, 40, 23
    cfg = dict(D=D, A=A, actor_h=[64, 48], critic_h=[64, 48], n_step=4, B=4, mode='clip', lr=1e-4, exp_interval=64,
               horizon=2, rnn_hidden=H, rnn_layer=1)
    lc, ec, sc = _rnn_cfg(cfg)
    ec.num_envs = N
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    gen = torch.Generator(device=DEV).manual_seed(N + H)
    u = lambda k, *s: (torch.rand(*s, generator=gen, device=DEV) * 2 - 1) * k  # noqa: E731
    k = 1.0 / H ** 0.5
    W = [u(k, 4 * H, D), u(k, 4 * H, H), u(k, 4 * H), u(k, 4 * H)]
    ag.model.rnn_stem.load_torch(dict(zip(['weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0'], W)))
    dims = [H, 64, 48, A]
    AL = [(u(dims[i] ** -0.5, dims[i + 1], dims[i]), u(dims[i] ** -0.5, dims[i + 1])) for i in range(3)]
    log_var = torch.full((A,), -1.0, device=DEV) + u(0.3, A)
    ag.model.actor.load_layers(AL, extra=log_var)
    zs = torch.cat([torch.randn(D, generator=gen, device=DEV) * 30, 300 * (1.5 + torch.rand(D, generator=gen, device=DEV)),
                    torch.tensor([300.0], device=DEV)])
    ag.model.z_stats.copy_(zs)
    noise = np.linspace(-0.3, 0.3, N)
    ag.set_noise(noise)
    W64, AL64 = [R.f64(w) for w in W], [(R.f64(w), R.f64(b)) for w, b in AL]
    sd64 = torch.exp(R.f64(log_var)[None] + torch.tensor(noise, dtype=torch.float64, device=DEV)[:, None])
    h64 = c64 = torch.zeros(N, H, dtype=torch.float64, device=DEV)
    rng = np.random.default_rng(N + H)
    worst = dict(pd=0.0, action=0.0, cells=0.0, drift=0.0)
    for t in range(steps):
        if t == reset_at:
            ag.reset()
            h64, c64 = torch.zeros_like(h64), torch.zeros_like(c64)
        h_prev, c_prev = [x.clone() for x in ag._rnn_state()]
        obs = torch.randn(N, D, generator=gen, device=DEV) * 1.5 + zs[:D] / 300.0
        eps = rng.standard_normal((N, A)).astype(np.float32)
        a, info = ag.act(obs, eps=eps)
        torch.cuda.synchronize()
        assert torch.equal(info[0][0][:, 0], h_prev) and torch.equal(info[0][1][:, 0], c_prev), 'onetime cells'
        if t in (0, reset_at):
            assert float(h_prev.abs().max()) == 0.0 and float(c_prev.abs().max()) == 0.0
        with torch.no_grad():
            x = R.zfilter(obs, zs)[:, None]
            r = R.lstm(x, R.f64(h_prev), R.f64(c_prev), *W64)
            mean = torch.tanh(R.trunk(r['h'][:, 0], AL64))
            act64 = torch.clamp(R.f64(eps).to(DEV) * sd64 + mean, -1.0, 1.0)
            e = dict(pd=float((info[1][0].double() - torch.cat([mean, sd64], 1)).abs().max()),
                     action=float((a.double() - act64).abs().max()),
                     cells=max(float((ag._h.double() - r['h_last']).abs().max()), float((ag._c.double() - r['c_last']).abs().max())))
            f = R.lstm(x, h64, c64, *W64)
            h64, c64 = f['h_last'], f['c_last']
            e['drift'] = max(float((ag._h.double() - h64).abs().max()), float((ag._c.double() - c64).abs().max()))
        for key, v in e.items():
            worst[key] = max(worst[key], v)
        assert max(e['pd'], e['action'], e['cells']) <= ACT_BAR, (t, e)
        assert e['drift'] <= DRIFT_BAR, (t, e)
    assert float(ag._c.abs().max()) > 0.3
    print('measured act', N, H, worst)


def test_default_ppo_config_runs_end_to_end():
    """BASELINE configs[0] stand-in: the UNMODIFIED PPO_DEFAULT_LEARNER_CONFIG (adapt mode + LSTM(100), n_step 25, stride 20,
    horizon 10, batch 64) on a synthetic 17-dim / 6-action env with the episode cap of 200: actors -> windows with the cells
    riding in the observation rows -> HBM FIFO -> learner.  The cells the learner reads for a window must be the cells the
    agent held at the window's first step, and learn() must agree with the RNN oracle on the same windows."""
    from surreal_b200.session import Config
    from surreal_b200.main.ppo_configs import (PPO_DEFAULT_LEARNER_CONFIG, PPO_DEFAULT_ENV_CONFIG, PPO_DEFAULT_SESSION_CONFIG,
                                               make_synthetic_env_config)
    from surreal_b200.agent import PPOAgent
    from surreal_b200.learner import PPOLearner
    from surreal_b200.replay import FIFOReplay
    from surreal_b200.env import SyntheticEnv
    from oracle.ppo_rnn import OraclePPOLearnerRNN
    from oracle.filters import ZFilter as OZ
    import tempfile
    lc = Config(copy.deepcopy(PPO_DEFAULT_LEARNER_CONFIG.to_dict()))
    ec = Config(copy.deepcopy(PPO_DEFAULT_ENV_CONFIG.to_dict()))
    sc = Config(copy.deepcopy(PPO_DEFAULT_SESSION_CONFIG.to_dict()))
    sc.folder = tempfile.mkdtemp()
    assert lc.algo.rnn.if_rnn_policy and lc.algo.ppo_mode == 'adapt'          # the reference's defaults, untouched
    N, D, A = 32, 17, 6            # 2 windows x 32 actors = one default batch of 64 (the default FIFO holds 96 + 3)
    make_synthetic_env_config(ec, N, D, A, seed=3)
    ec.limit_episode_length = 200
    n, stride, Hh, B = lc.algo.n_step, lc.algo.stride, lc.algo.rnn.rnn_hidden, lc.replay.batch_size
    R = FIFOReplay(lc, ec, sc)
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    env = SyntheticEnv(N, D, A, limit_episode_length=200, seed=3)
    ag.env = w = ag.prepare_env_agent(env)
    obs, _ = w.reset()
    cells_at = {}
    for t in range(n + stride):                                    # two (overlapping) windows per actor
        cells_at[t] = (ag._h.clone(), ag._c.clone())
        a = ag.act(obs)
        assert torch.equal(a[1][0][0][:, 0], cells_at[t][0])      # onetime_info = cells BEFORE the step
        obs, _, _, _ = w.step(a)
    torch.cuda.synchronize()
    assert len(R) == 2 * N == B
    L = PPOLearner(lc, ec, sc)
    L.model.load_state_dict(ag.model.state_dict())
    L.ref_target_model.update_target_params(L.model)
    b2 = R.sample(B)              # (step, actor) arrival order: rows 0..31 = first windows (cells: zeros), 32..63 = second ones
    h0, c0 = b2['onetime_infos'][0][:, 0], b2['onetime_infos'][1][:, 0]
    assert float(h0[:N].abs().max()) == 0.0 and float(c0[:N].abs().max()) == 0.0
    assert torch.equal(h0[N:], cells_at[stride][0]) and torch.equal(c0[N:], cells_at[stride][1])    # windows start at step `stride`
    assert float(h0[N:].abs().max()) > 0.0
    sd = {k: v.cpu() for k, v in L.model.state_dict().items()}
    al = [(sd['actor.model.seq.%d.weight' % (2 * i)], sd['actor.model.seq.%d.bias' % (2 * i)]) for i in range(3)]
    cl = [(sd['critic.model.seq.%d.weight' % (2 * i)], sd['critic.model.seq.%d.bias' % (2 * i)]) for i in range(3)]
    lstm = {k.split('.', 1)[1]: sd[k] for k in sd if k.startswith('rnn_stem.')}
    zf = OZ(D).load(sd['z_filter.running_sum'], sd['z_filter.running_sumsq'], sd['z_filter.count'])
    O = OraclePPOLearnerRNN(al, sd['actor.log_var'].view(1, A), cl, zf, lstm, A, n, B, lc.algo.rnn.horizon, Hh, 1, ppo_mode='adapt',
                            lr_actor=lc.algo.network.lr_actor, lr_critic=lc.algo.network.lr_critic)
    host = dict(obs=b2['obs']['low_dim']['flat_inputs'].cpu().numpy(), obs_next=b2['obs_next']['low_dim']['flat_inputs'].cpu().numpy(),
                actions=b2['actions'].cpu().numpy(), rewards=b2['rewards'].cpu().numpy(), dones=b2['dones'].cpu().numpy(),
                pd=b2['persistent_infos'][0].cpu().numpy(), h0=b2['onetime_infos'][0].cpu().numpy(), c0=b2['onetime_infos'][1].cpu().numpy())
    st = L.learn(b2)
    st_o = O.learn(host)
    torch.cuda.synchronize()
    assert L.last_n_policy_epochs == O.n_policy_epochs[-1]
    assert float((L._adv.cpu() - O.last_adv).abs().max()) <= 1e-5
    for k in ('_surr_loss', '_kl_loss_adapt', '_pol_kl', '_val_loss', '_entropy', '_avg_return_targ', '_avg_is_weight'):
        assert abs(st[k] - st_o[k]) <= 1e-5 * max(1.0, abs(st_o[k])), (k, st[k], st_o[k])

"""Stacked LSTM stems (algo.rnn.rnn_layer > 1) on the GPU: the stem's per-layer forward / BPTT against float64 autograd
over its shape envelope, PPOAgent.act against the reference golden and float64 steps at scale, PPOLearner.learn against
goldens the REAL reference produced at rnn_layer = 2 and 3, the cells' round trip through replay.insert / sample and a
host batch, the default config end to end, and checkpoints (ours and one the reference wrote)."""
import copy

import numpy as np
import pytest
import torch

from helpers import ppo_configs, ref_state_dict

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NAN = float('nan')
LOSS_STATS = ['_surr_loss', '_clip_surr_loss', '_kl_loss_adapt', '_entropy', '_pol_kl', '_val_loss', '_avg_return_targ',
              '_avg_log_sig', '_avg_behave_likelihood', '_avg_is_weight', '_ref_behave_diff', 'obs_running_mean',
              'obs_running_square', 'obs_running_std']


def _err(got, exp):
    e = (got.double() - exp).abs()
    return float(e.max()), float((got.double() - exp).norm()) / max(float(exp.norm()), 1e-30), \
        float(e.max()) / max(float(exp.abs().max()), 1e-30)


def _weights(gen, D, H, layers):
    k = 1.0 / H ** 0.5
    u = lambda *s: (torch.rand(*s, generator=gen, device=DEV) * 2 - 1) * k  # noqa: E731
    w = {}
    for l in range(layers):
        w.update({'weight_ih_l%d' % l: u(4 * H, D if l == 0 else H), 'weight_hh_l%d' % l: u(4 * H, H),
                  'bias_ih_l%d' % l: u(4 * H), 'bias_hh_l%d' % l: u(4 * H)})
    return w


# Bars per output; the worst error measured on an H100 80GB HBM3 (400 W power limit) over STACK_CASES is in the comment.
# Forward outputs are held to max |err|, dpre and the weight gradients to relative L2 and max |err| / max |g64|.
STACK_BAR = {'h': 3e-6,          # 4.0e-7 (h_out, h_prev, h_last of every layer)
             'gates': 8e-6,      # 1.1e-6
             'c': 6e-6,          # 9.6e-7 (c_seq, c_last)
             'dpre': 8e-6,       # 9.0e-7
             'dW': 7e-6}         # 7.3e-7 (dW_ih, dW_hh, db_ih, db_hh of every layer over 1..16 slabs)
# (B, T, D, H, layers, cells, splits).  cells: 'given' = one [L, B, H] tensor (then also run in place, as the agent does),
# 'none' = zeros, 'wide' = per-layer views into wider NaN-filled record rows (ld_cells = the row stride, as the learner reads them)
STACK_CASES = [(1, 1, 1, 1, 3, 'given', 1), (3, 2, 5, 7, 2, 'none', 2), (6, 26, 3, 31, 2, 'wide', 1),
               (64, 26, 17, 100, 2, 'wide', 16), (5, 29, 9, 100, 3, 'given', 3), (4096, 2, 33, 256, 2, 'wide', 16),
               (16, 30, 17, 256, 3, 'given', 7), (1024, 1, 17, 100, 2, 'none', 8), (64, 16, 17, 100, 3, 'wide', 5)]


@pytest.mark.parametrize('B,T,D,H,layers,cells,splits', STACK_CASES)
def test_stacked_stem_matches_float64(B, T, D, H, layers, cells, splits):
    """LSTMStem / RnnTrainer with 2 or 3 layers against lstm_stack (grad_ref_stacked) in float64: every layer's h_out, h_prev,
    gates, c_seq, dpre, last cells and its four weight / bias gradients.  NaN sentinels in the padding columns of every
    layer's h_out / h_prev and in the record rows around the cells must stay untouched."""
    import grad_ref as R
    from grad_ref_stacked import lstm_stack
    from surreal_b200.model.lstm_stem import LSTMStem, RnnTrainer
    from surreal_b200.utils import CellLayout
    gen = torch.Generator(device=DEV).manual_seed(B * 7 + T * 3 + H + layers)
    w = _weights(gen, D, H, layers)
    stem = LSTMStem(D, H, DEV, layers=layers)
    stem.load_torch(w)
    Rn, Hp = B * T, (H + 3) // 4 * 4
    h64 = c64 = None
    ld, rows = H, None
    if cells == 'none':
        h0 = c0 = None
        ld = 0
    else:
        hs = torch.randn(layers, B, H, generator=gen, device=DEV) * 0.5
        cs = torch.randn(layers, B, H, generator=gen, device=DEV) * 0.8
        h64, c64 = list(hs.double()), list(cs.double())
        if cells == 'given':
            h0, c0 = hs.clone(), cs.clone()
        else:
            cl = CellLayout(layers, H, D)
            rows = torch.full((B, 26, cl.width), NAN, device=DEV)
            for k in range(layers):
                cl.h(rows[:, 0], k).copy_(hs[k])
                cl.c(rows[:, 0], k).copy_(cs[k])
            h0 = [cl.h(rows[:, 0], k) for k in range(layers)]
            c0 = [cl.c(rows[:, 0], k) for k in range(layers)]
            ld = rows.stride(0)
            rows_before = rows.clone()
    x = torch.randn(B, T, D, generator=gen, device=DEV)
    xf = torch.zeros(Rn, (D + 3) // 4 * 4, device=DEV)[:, :D]
    xf.copy_(x.reshape(Rn, D))
    tr = RnnTrainer(stem, B, T, splits=splits)
    for k in range(layers):
        for name in ('h_out', 'h_prev'):
            tr.bufs[name + ('' if k == 0 else str(k))] = torch.full((Rn, Hp), NAN, device=DEV)[:, :H]
    h_top = tr.forward(xf, h0, c0, ld)
    dout = torch.randn(B, T, H, generator=gen, device=DEV)
    dh = torch.full((Rn, Hp + 4), NAN, device=DEV)
    dh[:, :H] = dout.reshape(Rn, H)
    tr.backward(dh)
    torch.cuda.synchronize()
    if rows is not None:
        assert torch.equal(rows.nan_to_num(7.0), rows_before.nan_to_num(7.0)), 'record rows written'
    names = [['weight_ih_l%d' % k, 'weight_hh_l%d' % k, 'bias_ih_l%d' % k, 'bias_hh_l%d' % k] for k in range(layers)]
    W = [[R.f64(w[n]).requires_grad_(True) for n in ns] for ns in names]
    rs = lstm_stack(R.f64(x), h64, c64, W)
    seed = R.f64(dout)
    flatW = [p for ws in W for p in ws]
    pres = [p for r in rs for p in r['pre']]
    gs = torch.autograd.grad((rs[-1]['h'] * seed).sum(), flatW + pres)
    worst = {}

    def fwd(name, got, exp):
        e = _err(got, exp)[0]
        worst[name] = max(worst.get(name, 0.0), e)
        assert e <= STACK_BAR[name], (name, e)

    def rel(name, got, exp):
        _, r_, m_ = _err(got, exp)
        worst[name] = max(worst.get(name, 0.0), r_, m_)
        assert r_ <= STACK_BAR[name] and m_ <= STACK_BAR[name], (name, r_, m_)

    assert h_top.data_ptr() == stem.layer_bufs(tr.bufs, layers - 1)['h_out'].data_ptr()
    g = tr.slabs.double().sum(0).float()
    for k in range(layers):
        lb = stem.layer_bufs(tr.bufs, k)
        for name in ('h_out', 'h_prev'):
            assert bool(torch.isnan(lb[name]._base[:, H:]).all()), ('padding written', name, k)
        hk0 = h64[k] if h64 is not None else torch.zeros(B, H, dtype=torch.float64, device=DEV)
        fwd('h', lb['h_out'], rs[k]['h'].detach().reshape(Rn, H))
        fwd('h', lb['h_prev'], torch.cat([hk0[:, None], rs[k]['h'].detach()[:, :-1]], 1).reshape(Rn, H))
        fwd('gates', lb['gates'], rs[k]['gates'].detach().reshape(Rn, 4 * H))
        fwd('c', lb['c_seq'], rs[k]['c'].detach().reshape(Rn, H))
        dpre_ref = torch.stack(gs[4 * layers + k * T:4 * layers + (k + 1) * T], 1).reshape(Rn, 4 * H)
        rel('dpre', tr.dpres[k], dpre_ref)
        sfx = '' if k == 0 else str(k)
        o_i, n_i = stem.off['ih' + sfx]
        o_h, n_h = stem.off['hh' + sfx]
        wi, bi = stem.ihs[k].get_layer(0, g[o_i:o_i + n_i])
        wh, bh = stem.hhs[k].get_layer(0, g[o_h:o_h + n_h])
        for got, exp in ((wi, gs[4 * k]), (wh, gs[4 * k + 1]), (bi, gs[4 * k + 2]), (bh, gs[4 * k + 3])):
            rel('dW', got, exp)
    # last cells of every layer, into their own [L, B, H] buffers and (given cells) in place over the initial cells
    bufs = stem.buffers(B, T, save=False)
    hl, cl_ = torch.full((layers, B, H), NAN, device=DEV), torch.full((layers, B, H), NAN, device=DEV)
    out = stem.forward(xf, h0, c0, ld, B, T, bufs, h_last=hl, c_last=cl_)
    torch.cuda.synchronize()
    assert torch.equal(out, h_top), 'the forward without saves differs'
    for k in range(layers):
        fwd('h', hl[k], rs[k]['h_last'].detach())
        fwd('c', cl_[k], rs[k]['c_last'].detach())
    if cells == 'given':
        stem.forward(xf, h0, c0, ld, B, T, bufs, h_last=h0, c_last=c0)
        torch.cuda.synchronize()
        assert torch.equal(h0, hl) and torch.equal(c0, cl_), 'in-place update differs'
    print('measured stack', B, T, D, H, layers, cells, worst)


def test_stem_state_dict_names_and_offsets():
    """rnn_stem.{weight,bias}_{ih,hh}_l{k}: torch's names and shapes; segments ih_0, hh_0, ih_1, hh_1 in the flat buffer,
    layer 0 at the offsets of the one-layer stem; load_torch / state_items round trip every layer."""
    from surreal_b200.model.lstm_stem import LSTMStem
    D, H = 13, 9
    one, three = LSTMStem(D, H, DEV), LSTMStem(D, H, DEV, layers=3)
    assert three.off['ih'] == one.off['ih'] and three.off['hh'] == one.off['hh']
    assert three.off['ih1'][0] == one.size and three.off['hh2'][0] + three.off['hh2'][1] == three.size
    ref = torch.nn.LSTM(D, H, 3, batch_first=True)
    sd = {k: v.detach() for k, v in ref.state_dict().items()}
    three.load_torch(sd, prefix='')
    items = dict(three.state_items())
    assert sorted(items) == sorted('rnn_stem.' + k for k in sd)
    for k, v in sd.items():
        assert torch.equal(items['rnn_stem.' + k].cpu(), v), k
    assert tuple(items['rnn_stem.weight_ih_l1'].shape) == (4 * H, H)


def _rnn_cfg(cfg, B=None):
    lc, ec, sc = ppo_configs(D=cfg['D'], A=cfg['A'], actor_h=cfg['actor_h'], critic_h=cfg['critic_h'], n_step=cfg['n_step'],
                             stride=cfg['n_step'], B=B or cfg['B'], mode=cfg['mode'], lr=cfg['lr'], exp_interval=cfg['exp_interval'])
    lc.algo.rnn.if_rnn_policy = True
    lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = cfg['horizon'], cfg['rnn_hidden'], cfg['rnn_layer']
    return lc, ec, sc


def _host_batch(b):
    return {'obs': {'low_dim': {'flat_inputs': b['obs']}}, 'obs_next': {'low_dim': {'flat_inputs': b['obs_next']}},
            'actions': b['actions'], 'rewards': b['rewards'], 'dones': b['dones'], 'persistent_infos': [b['pd']],
            'onetime_infos': [b['h0'], b['c0']]}


@pytest.mark.parametrize('tag', ['rnn2_clip', 'rnn2_adapt', 'rnn3_clip'])
def test_ppo_learn_stacked_matches_reference(golden, tag):
    """learn() + publish_parameter with 2 / 3 LSTM layers against the reference: advantages, returns and statistics within
    1e-5, the same KL early-stop epoch and clip_epsilon / beta path, every parameter (all layers of the stem)."""
    from surreal_b200.learner import PPOLearner
    g = golden('ppo_learn_' + tag)
    cfg, hyper, stats = g.js('cfg'), g.js('hyper'), g.js('stats')
    lc, ec, sc = _rnn_cfg(cfg)
    L = PPOLearner(lc, ec, sc)
    assert L.model.rnn_stem.layers == cfg['rnn_layer']
    L.model.load_state_dict(ref_state_dict(g.sub('init/')))
    L.ref_target_model.update_target_params(L.model)
    lr, E = cfg['lr'], cfg['n_step'] - cfg['horizon'] + 1
    for it in range(cfg['iters']):
        b = g.sub('it%d/' % it)
        st = L.learn(_host_batch(b))
        L.publish_parameter(it, message='')
        torch.cuda.synchronize()
        assert L._adv.shape == (cfg['B'], E)
        assert float((L._adv.cpu() - torch.tensor(b['adv'])).abs().max()) <= 1e-5
        rms = float(np.sqrt((b['ret'] ** 2).mean()))
        assert float((L._ret.cpu() - torch.tensor(b['ret'])).abs().max()) <= 1e-5 * max(1.0, rms)
        assert L.last_n_policy_epochs == hyper[it]['n_policy_epochs'], 'KL early stop diverged'
        for k, v in stats[it].items():
            tol = 1e-5 * max(1.0, abs(v)) if k in LOSS_STATS else 2e-4 * max(1.0, abs(v))
            if k == '_val_explained_var':
                tol = 1e-4
            assert abs(st[k] - v) <= tol, '%s it%d: got %.9g expected %.9g' % (k, it, st[k], v)
        after = ref_state_dict(g.sub('it%d/after/' % it))
        got = L.model.state_dict()
        assert set(after) == set(got), sorted(set(after) ^ set(got))
        worst = 0.0
        for k, e in after.items():
            gk = got[k].cpu().reshape(e.shape)
            if k.startswith('z_filter'):
                assert float((gk - e).abs().max()) <= 1e-6 * max(1.0, float(e.abs().max())), k
                continue
            worst = max(worst, float((gk - e).abs().max()))
        print('measured params', tag, it, worst)
        assert worst <= max(2e-6, 0.02 * lr), 'params drifted by %.3e' % worst
        if cfg['mode'] == 'clip':
            assert L.clip_epsilon == pytest.approx(hyper[it]['clip_epsilon'], rel=1e-12)
        else:
            assert L.beta == pytest.approx(hyper[it]['beta'], rel=1e-12)
        assert L.exp_counter == hyper[it]['exp_counter']


def _snapshot(L):
    m = L.model
    return [m.actor.params, m.critic.params, m.rnn_stem.params, m.z_stats, L.actor_rnn.exp_avg, L.actor_rnn.exp_avg_sq,
            L.critic_rnn.exp_avg, L.critic_rnn.exp_avg_sq, L.actor_optim.exp_avg_sq, L.critic_optim.exp_avg_sq,
            L.ref_target_model.rnn_stem.params]


@pytest.mark.parametrize('tag', ['rnn2_clip', 'rnn2_adapt'])
def test_graph_and_eager_learn_are_bit_identical(golden, tag):
    from surreal_b200.learner import PPOLearner
    g = golden('ppo_learn_' + tag)
    cfg = g.js('cfg')
    runs = []
    for graph in (True, False):
        lc, ec, sc = _rnn_cfg(cfg)
        L = PPOLearner(lc, ec, sc)
        L.use_cuda_graph = graph
        L.model.load_state_dict(ref_state_dict(g.sub('init/')))
        L.ref_target_model.update_target_params(L.model)
        sts = []
        for it in range(cfg['iters']):
            sts.append(L.learn(_host_batch(g.sub('it%d/' % it))))
            L.publish_parameter(it, message='')
        torch.cuda.synchronize()
        runs.append((sts, [t.clone() for t in _snapshot(L)]))
    assert runs[0][0] == runs[1][0]
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)


def _agent(N, D, A, H, layers, actor_h=(64, 48), critic_h=(64, 48)):
    from surreal_b200.agent import PPOAgent
    cfg = dict(D=D, A=A, actor_h=list(actor_h), critic_h=list(critic_h), n_step=4, B=4, mode='clip', lr=1e-4, exp_interval=64,
               horizon=2, rnn_hidden=H, rnn_layer=layers)
    lc, ec, sc = _rnn_cfg(cfg)
    ec.num_envs = N
    return PPOAgent(lc, ec, sc, 0, 'training')


def test_ppo_agent_act_rnn2_matches_reference(golden):
    """One actor with a 2-layer LSTM, seven steps: numpy in, onetime_infos (2, H) = the cells BEFORE the step, reset()."""
    g = golden('ppo_act_rnn2')
    Hd = int(g['rnn_hidden'])
    ag = _agent(1, 11, 3, Hd, 2, actor_h=(32, 24), critic_h=(28, 20))
    ag.model.load_state_dict(ref_state_dict(g.sub('model/')))
    ag.set_noise(np.array([float(g['noise'])]))
    for i in range(len(g['obs'])):
        if i == int(g['reset_at']):
            ag.reset()
        a, info = ag.act(g['obs'][i], eps=g['eps'][i])
        assert info[0][0].shape == (2, Hd) and info[0][1].shape == (2, Hd)
        np.testing.assert_allclose(info[0][0], g['h_before'][i], rtol=0, atol=2e-6)
        np.testing.assert_allclose(info[0][1], g['c_before'][i], rtol=0, atol=2e-6)
        np.testing.assert_allclose(info[1][0], g['pds'][i], rtol=0, atol=2e-6)
        np.testing.assert_allclose(a, g['actions'][i], rtol=0, atol=5e-6)


ACT_BAR = 2.5e-6      # one step from the agent's own cells: pd, action and every layer's new cells; measured 2.7e-7
DRIFT_BAR = 1.5e-6    # free-running float64 trajectory against the agent's cells over 40 steps; measured 1.7e-7


@pytest.mark.parametrize('N,H,layers', [(1, 100, 2), (64, 256, 3), (1024, 100, 2), (1024, 256, 3), (1024, 100, 3)])
def test_ppo_agent_act_stacked_at_scale(N, H, layers):
    """40 steps with injected eps, per-actor noise and a reset() at step 23.  Every step: onetime_infos [N, L, H] are
    exactly the cells held before the step; pd, the action and every layer's cells (updated in place) match one float64
    step of the stacked LSTM taken from those cells; the free-running float64 trajectory stays within DRIFT_BAR."""
    import grad_ref as R
    from grad_ref_stacked import lstm_stack
    D, A, steps, reset_at = 17, 6, 40, 23
    ag = _agent(N, D, A, H, layers)
    gen = torch.Generator(device=DEV).manual_seed(N + H + layers)
    u = lambda k, *s: (torch.rand(*s, generator=gen, device=DEV) * 2 - 1) * k  # noqa: E731
    w = _weights(gen, D, H, layers)
    ag.model.rnn_stem.load_torch(w)
    dims = [H, 64, 48, A]
    AL = [(u(dims[i] ** -0.5, dims[i + 1], dims[i]), u(dims[i] ** -0.5, dims[i + 1])) for i in range(3)]
    log_var = torch.full((A,), -1.0, device=DEV) + u(0.3, A)
    ag.model.actor.load_layers(AL, extra=log_var)
    zs = torch.cat([torch.randn(D, generator=gen, device=DEV) * 30, 300 * (1.5 + torch.rand(D, generator=gen, device=DEV)),
                    torch.tensor([300.0], device=DEV)])
    ag.model.z_stats.copy_(zs)
    noise = np.linspace(-0.3, 0.3, N)
    ag.set_noise(noise)
    W64 = [[R.f64(w['%s_l%d' % (n, k)]) for n in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')] for k in range(layers)]
    AL64 = [(R.f64(a), R.f64(b)) for a, b in AL]
    sd64 = torch.exp(R.f64(log_var)[None] + torch.tensor(noise, dtype=torch.float64, device=DEV)[:, None])
    z64 = torch.zeros(layers, N, H, dtype=torch.float64, device=DEV)
    h64, c64 = z64.clone(), z64.clone()
    rng = np.random.default_rng(N + H)
    worst = dict(pd=0.0, action=0.0, cells=0.0, drift=0.0)
    for t in range(steps):
        if t == reset_at:
            ag.reset()
            h64, c64 = z64.clone(), z64.clone()
        h_prev, c_prev = [x.clone() for x in ag._rnn_state()]
        assert tuple(h_prev.shape) == (layers, N, H)
        obs = torch.randn(N, D, generator=gen, device=DEV) * 1.5 + zs[:D] / 300.0
        eps = rng.standard_normal((N, A)).astype(np.float32)
        a, info = ag.act(obs, eps=eps)
        torch.cuda.synchronize()
        assert tuple(info[0][0].shape) == (N, layers, H)
        assert torch.equal(info[0][0], h_prev.transpose(0, 1)) and torch.equal(info[0][1], c_prev.transpose(0, 1)), 'onetime cells'
        if t in (0, reset_at):
            assert float(h_prev.abs().max()) == 0.0 and float(c_prev.abs().max()) == 0.0
        with torch.no_grad():
            x = R.zfilter(obs, zs)[:, None]
            rs = lstm_stack(x, list(R.f64(h_prev)), list(R.f64(c_prev)), W64)
            mean = torch.tanh(R.trunk(rs[-1]['h'][:, 0], AL64))
            act64 = torch.clamp(R.f64(eps).to(DEV) * sd64 + mean, -1.0, 1.0)
            e = dict(pd=float((info[1][0].double() - torch.cat([mean, sd64], 1)).abs().max()),
                     action=float((a.double() - act64).abs().max()),
                     cells=max(max(float((ag._hs[k].double() - rs[k]['h_last']).abs().max()),
                                   float((ag._cs[k].double() - rs[k]['c_last']).abs().max())) for k in range(layers)))
            f = lstm_stack(x, list(h64), list(c64), W64)
            h64 = torch.stack([r['h_last'] for r in f])
            c64 = torch.stack([r['c_last'] for r in f])
            e['drift'] = max(float((ag._hs.double() - h64).abs().max()), float((ag._cs.double() - c64).abs().max()))
        for key, v in e.items():
            worst[key] = max(worst[key], v)
        assert max(e['pd'], e['action'], e['cells']) <= ACT_BAR, (t, e)
        assert e['drift'] <= DRIFT_BAR, (t, e)
    assert float(ag._cs[layers - 1].abs().max()) > 0.1
    print('measured act', N, H, layers, worst)


@pytest.mark.parametrize('layers', [1, 2, 3])
def test_onetime_infos_shapes(layers):
    """onetime_infos: [N, L, H] for device tensors and numpy batches, [L, H] for one actor with a 1-D observation."""
    D, A, H = 7, 2, 5
    for N in (4, 1):
        ag = _agent(N, D, A, H, layers, actor_h=(8, 8))
        for k in range(3):
            _, info = ag.act(torch.randn(N, D, device=DEV))
            assert isinstance(info[0][0], torch.Tensor) and tuple(info[0][0].shape) == (N, layers, H)
            _, info = ag.act(np.random.default_rng(k).standard_normal((N, D)).astype(np.float32))
            exp = (layers, H) if N == 1 else (N, layers, H)
            assert isinstance(info[0][0], np.ndarray) and info[0][0].shape == exp and info[0][1].shape == exp
        if N == 1:
            _, info = ag.act(np.zeros(D, dtype=np.float32))
            assert info[0][0].shape == (layers, H)
        np.testing.assert_array_equal(info[0][0], ag._hs_before.cpu().numpy().transpose(1, 0, 2).reshape(info[0][0].shape))


def _window(rng, n, D, A, layers, H):
    obs = [{'low_dim': {'flat_inputs': rng.standard_normal(D).astype(np.float32)}} for _ in range(n)]
    nxt = {'low_dim': {'flat_inputs': rng.standard_normal(D).astype(np.float32)}}
    pinfo = [[rng.standard_normal(2 * A).astype(np.float32)] for _ in range(n)]
    hc = [rng.standard_normal((layers, H)).astype(np.float32), rng.standard_normal((layers, H)).astype(np.float32)]
    return ({'obs': obs, 'obs_next': nxt},
            {'actions': [rng.standard_normal(A) for _ in range(n)], 'onetime_infos': hc, 'persistent_infos': pinfo,
             'rewards': [float(r) for r in rng.standard_normal(n)], 'dones': [False] * n, 'infos': [{}] * n, 'n_step': n})


@pytest.mark.parametrize('layers', [2, 3])
def test_cells_round_trip_through_replay_and_learner(layers):
    """Reference-shaped windows (onetime_infos [L, H]) through the experience wire and replay.insert come back from
    sample() bit-exact as [B, L, H]; the same cells as a numpy batch land bit-exact in the learner's rows.  A window whose
    cells have the wrong size is rejected."""
    from surreal_b200 import exp_wire as W
    from surreal_b200.learner import PPOLearner
    from surreal_b200.replay import FIFOReplay
    n, D, A, H, B = 5, 6, 2, 9, 8
    lc, ec, sc = ppo_configs(D=D, A=A, n_step=n, stride=n, B=B, memory_size=32)
    lc.algo.rnn.if_rnn_policy = True
    lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = 2, H, layers
    Rp = FIFOReplay(lc, ec, sc)
    rng = np.random.default_rng(layers)
    wins = [_window(rng, n, D, A, layers, H) for _ in range(B)]
    buf = W.ExpBuffer()
    for h, nn in wins:
        buf.add(h, nn)
    for exp in W.inflate(buf.flush()):
        Rp.insert(exp)
    assert len(Rp) == B
    b = Rp.sample(B)
    torch.cuda.synchronize()
    h0, c0 = b['onetime_infos']
    assert tuple(h0.shape) == (B, layers, H) and tuple(c0.shape) == (B, layers, H)
    exp_h = np.stack([nn['onetime_infos'][0] for _, nn in wins])
    exp_c = np.stack([nn['onetime_infos'][1] for _, nn in wins])
    np.testing.assert_array_equal(h0.cpu().numpy(), exp_h)
    np.testing.assert_array_equal(c0.cpu().numpy(), exp_c)
    np.testing.assert_array_equal(b['obs']['low_dim']['flat_inputs'][:, 0].cpu().numpy(),
                                  np.stack([h['obs'][0]['low_dim']['flat_inputs'] for h, _ in wins]))
    # the device batch and the same windows as a numpy batch give the learner the same rows
    L = PPOLearner(lc, ec, sc)
    L.learn(b)
    torch.cuda.synchronize()
    dev_rows = L._obs_full.clone()
    host = {'obs': {'low_dim': {'flat_inputs': b['obs']['low_dim']['flat_inputs'].cpu().numpy()}},
            'obs_next': {'low_dim': {'flat_inputs': b['obs_next']['low_dim']['flat_inputs'].cpu().numpy()}},
            'actions': b['actions'].cpu().numpy(), 'rewards': b['rewards'].cpu().numpy(), 'dones': b['dones'].cpu().numpy(),
            'persistent_infos': [b['persistent_infos'][0].cpu().numpy()], 'onetime_infos': [exp_h, exp_c]}
    L2 = PPOLearner(lc, ec, sc)
    L2.learn(host)
    torch.cuda.synchronize()
    cl = L2.cell_layout
    np.testing.assert_array_equal(cl.h(L2._obs_full[:, 0]).cpu().numpy().reshape(B, layers, H), exp_h)
    np.testing.assert_array_equal(cl.c(L2._obs_full[:, 0]).cpu().numpy().reshape(B, layers, H), exp_c)
    assert torch.equal(L2._obs_full[:, 0], dev_rows[:, 0])
    h, nn = _window(rng, n, D, A, layers, H)
    nn['onetime_infos'] = [nn['onetime_infos'][0][:1], nn['onetime_infos'][1][:1]]      # one layer's cells only
    with pytest.raises(ValueError):
        Rp.insert(dict(h, **nn))


def test_default_config_with_two_layers_end_to_end():
    """The UNMODIFIED default PPO config with rnn_layer = 2: actors (device env behind the window wrapper) -> FIFO ->
    learner.  Every stored window's row-0 cells equal the agent's cells at the window's first step, and learn() agrees
    with the RNN oracle on the same windows."""
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
    lc.algo.rnn.rnn_layer = 2
    N, D, A = 32, 17, 6
    make_synthetic_env_config(ec, N, D, A, seed=3)
    ec.limit_episode_length = 200
    n, stride, Hh, B = lc.algo.n_step, lc.algo.stride, lc.algo.rnn.rnn_hidden, lc.replay.batch_size
    R = FIFOReplay(lc, ec, sc)
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    env = SyntheticEnv(N, D, A, limit_episode_length=200, seed=3)
    ag.env = w = ag.prepare_env_agent(env)
    obs, _ = w.reset()
    cells_at = {}
    for t in range(n + stride):
        cells_at[t] = (ag._hs.clone(), ag._cs.clone())
        a = ag.act(obs)
        assert torch.equal(a[1][0][0], cells_at[t][0].transpose(0, 1))
        obs, _, _, _ = w.step(a)
    torch.cuda.synchronize()
    assert len(R) == 2 * N == B
    L = PPOLearner(lc, ec, sc)
    L.model.load_state_dict(ag.model.state_dict())
    L.ref_target_model.update_target_params(L.model)
    b2 = R.sample(B)
    h0, c0 = b2['onetime_infos']
    assert tuple(h0.shape) == (B, 2, Hh)
    assert float(h0[:N].abs().max()) == 0.0 and float(c0[:N].abs().max()) == 0.0
    assert torch.equal(h0[N:], cells_at[stride][0].transpose(0, 1)) and torch.equal(c0[N:], cells_at[stride][1].transpose(0, 1))
    assert float(h0[N:, 1].abs().max()) > 0.0 and not torch.equal(h0[N:, 0], h0[N:, 1])
    sd = {k: v.cpu() for k, v in L.model.state_dict().items()}
    al = [(sd['actor.model.seq.%d.weight' % (2 * i)], sd['actor.model.seq.%d.bias' % (2 * i)]) for i in range(3)]
    cl = [(sd['critic.model.seq.%d.weight' % (2 * i)], sd['critic.model.seq.%d.bias' % (2 * i)]) for i in range(3)]
    lstm = {k.split('.', 1)[1]: sd[k] for k in sd if k.startswith('rnn_stem.')}
    assert 'weight_hh_l1' in lstm
    zf = OZ(D).load(sd['z_filter.running_sum'], sd['z_filter.running_sumsq'], sd['z_filter.count'])
    O = OraclePPOLearnerRNN(al, sd['actor.log_var'].view(1, A), cl, zf, lstm, A, n, B, lc.algo.rnn.horizon, Hh, 2, ppo_mode='adapt',
                            lr_actor=lc.algo.network.lr_actor, lr_critic=lc.algo.network.lr_critic)
    host = dict(obs=b2['obs']['low_dim']['flat_inputs'].cpu().numpy(), obs_next=b2['obs_next']['low_dim']['flat_inputs'].cpu().numpy(),
                actions=b2['actions'].cpu().numpy(), rewards=b2['rewards'].cpu().numpy(), dones=b2['dones'].cpu().numpy(),
                pd=b2['persistent_infos'][0].cpu().numpy(), h0=h0.cpu().numpy(), c0=c0.cpu().numpy())
    st = L.learn(b2)
    st_o = O.learn(host)
    torch.cuda.synchronize()
    assert L.last_n_policy_epochs == O.n_policy_epochs[-1]
    assert float((L._adv.cpu() - O.last_adv).abs().max()) <= 1e-5
    for k in ('_surr_loss', '_kl_loss_adapt', '_pol_kl', '_val_loss', '_entropy', '_avg_return_targ', '_avg_is_weight'):
        assert abs(st[k] - st_o[k]) <= 1e-5 * max(1.0, abs(st_o[k])), (k, st[k], st_o[k])


def test_stacked_learner_checkpoint_roundtrip(tmp_path, golden):
    """A 2-layer learner saved with its optimiser state (heads and both optimisers' stem Adam moments) and restored
    continues bit-identically."""
    from surreal_b200.learner import PPOLearner
    g = golden('ppo_learn_rnn2_clip')
    cfg = g.js('cfg')

    def make(folder, restore_from=None):
        lc, ec, sc = _rnn_cfg(cfg)
        sc.folder = str(folder)
        sc.checkpoint.learner.periodic = 1
        sc.checkpoint.learner.min_interval = 0
        sc.checkpoint.learner.include_optimizer = True
        if restore_from is not None:
            sc.checkpoint.restore = True
            sc.checkpoint.restore_folder = str(restore_from)
        return PPOLearner(lc, ec, sc)
    torch.manual_seed(5)
    A_ = make(tmp_path / 'a')
    for it in range(2):
        A_.learn(_host_batch(g.sub('it%d/' % it)))
        if it < 1:
            A_.publish_parameter(it)
    torch.manual_seed(555)
    B_ = make(tmp_path / 'b', restore_from=tmp_path / 'a')
    for k, v in A_.model.state_dict().items():
        assert torch.equal(v, B_.model.state_dict()[k]), k
    assert 'rnn_stem.weight_ih_l1' in A_.model.state_dict()
    nxt = _host_batch(g.sub('it2/'))
    sa, sb = A_.learn(nxt), B_.learn(nxt)
    torch.cuda.synchronize()
    assert sa == sb
    for a, b in zip(_snapshot(A_), _snapshot(B_)):
        assert torch.equal(a, b)


def test_reference_written_stacked_checkpoint_restores(tmp_path, golden):
    """The folder in tests/golden/ppo_learner_ckpt_rnn2.npz was written by the reference's PeriodicCheckpoint for a real
    reference PPOLearner with a 2-layer LSTM: it restores into PPOLearner with every layer's parameters."""
    from surreal_b200.learner import PPOLearner
    g = golden('ppo_learner_ckpt_rnn2')
    cfg = g.js('cfg')
    ck = tmp_path / 'ref' / 'checkpoint'
    ck.mkdir(parents=True)
    names = g.js('file_names') if g['file_names'].ndim == 0 else [str(x) for x in g['file_names']]
    for fn in names:
        (ck / fn).write_bytes(bytes(g['file/' + fn]))
    lc, ec, sc = _rnn_cfg(dict(cfg, mode='clip'))
    sc.folder = str(tmp_path / 'mine')
    sc.checkpoint.restore = True
    sc.checkpoint.restore_folder = str(tmp_path / 'ref')
    L = PPOLearner(lc, ec, sc)
    assert L.current_iteration == cfg['current_iteration']
    for name, model in (('saved/model/', L.model), ('saved/ref/', L.ref_target_model)):
        exp = ref_state_dict(g.sub(name))
        assert 'rnn_stem.bias_hh_l1' in exp
        got = model.state_dict()
        assert set(exp) == set(got)
        for k, e in exp.items():
            assert torch.equal(got[k].cpu().reshape(e.shape), e), k
    L.learn(_random_batch(cfg))                                     # and it trains
    torch.cuda.synchronize()


def _random_batch(cfg):
    rng = np.random.default_rng(0)
    B, n, D, A, H, Lr = cfg['B'], cfg['n_step'], cfg['D'], cfg['A'], cfg['rnn_hidden'], cfg['rnn_layer']
    pd = np.concatenate([np.tanh(rng.standard_normal((B, n, A))) * 0.5, np.full((B, n, A), 0.4)], -1).astype(np.float32)
    return {'obs': {'low_dim': {'flat_inputs': rng.standard_normal((B, n, D)).astype(np.float32)}},
            'obs_next': {'low_dim': {'flat_inputs': rng.standard_normal((B, 1, D)).astype(np.float32)}},
            'actions': np.clip(rng.standard_normal((B, n, A)) * 0.4, -1, 1), 'rewards': rng.standard_normal((B, n)),
            'dones': np.zeros((B, n), np.float32), 'persistent_infos': [pd],
            'onetime_infos': [rng.standard_normal((B, Lr, H)).astype(np.float32) * 0.1,
                              rng.standard_normal((B, Lr, H)).astype(np.float32) * 0.1]}

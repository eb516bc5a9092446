"""RNN mode's learner gradients against float64 autograd (tests/grad_ref.py ppo_policy_rnn / value_rnn).

In RNN mode each optimiser steps ONE gradient over [head | LSTM stem] (model/cnn_stem.py joint_step), with its own Adam
state for the shared stem, and the value epochs run on the stem the policy epochs have already stepped.  These tests read
those gradients (PPOLearner._g_actor / _g_critic) in eager learn() calls whose epochs are wrapped to snapshot the
parameters each epoch starts from, and compare them with float64 autograd on the batch's own initial cells, the z-filter
statistics before learn(), the learner's own advantages / returns and the reference policy.  Every bar quotes the worst
ratio measured on an H100 80GB HBM3 next to it."""
import copy
import math

import numpy as np
import pytest
import torch

import grad_ref as R
from helpers import ppo_configs

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
# Each bar is followed by the worst value measured over these tests.
RNN_LEARN_BAR = 5e-5  # [head | stem] gradients per tensor, relative L2 and max error / max|g64|: 5.7e-6 (the
                      # third policy epoch); 2.6e-6 for one epoch (big_clip: 16k rows over 16 slabs)
GN_BAR = 1e-5         # joint gradient norms, relative: 1.5e-6
MOMENT_BAR = 1e-6     # each optimiser's stem Adam moments against (1 - beta) g' (and g'^2), relative L2: 1.2e-7
VALUE_BAR = 1e-5      # critic pass over all B (n + 1) rows, max error / max|v64|: 2.4e-6
GAE_BAR = 5e-6        # advantages (normalised), max error: 5.9e-7; returns, max error / max(1, rms): 3.6e-7
ZF_BAR = 5e-7         # z-filter sums after learn(), max error / max|sum|: 7.4e-8

# name: D, A, actor / critic hidden, n_step, horizon, rnn_hidden, batch, mode.  'default' is the unmodified
# PPO_DEFAULT_LEARNER_CONFIG (17-dim observations, 6 actions) with one epoch of each optimiser.
CASES = {
    'default': dict(default=True, D=17, A=6),
    'big_clip': dict(D=64, A=8, actor_h=(256, 256), critic_h=(256, 256), n=25, horizon=10, H=100, B=1024, mode='clip'),
    'h256_full_bptt': dict(D=17, A=6, actor_h=(64, 48), critic_h=(64, 48), n=25, horizon=1, H=256, B=64, mode='adapt-hinge'),
    'eff_len_1': dict(D=11, A=3, actor_h=(32, 24), critic_h=(28, 20), n=8, horizon=8, H=100, B=256, mode='clip'),
}


def _configs(c, epoch_policy=1, lr=None):
    if c.get('default'):
        from surreal_b200.session import Config
        from surreal_b200.main.ppo_configs import (PPO_DEFAULT_LEARNER_CONFIG, PPO_DEFAULT_ENV_CONFIG,
                                                   PPO_DEFAULT_SESSION_CONFIG)
        import tempfile
        lc = Config(copy.deepcopy(PPO_DEFAULT_LEARNER_CONFIG.to_dict()))
        ec = Config(copy.deepcopy(PPO_DEFAULT_ENV_CONFIG.to_dict()))
        sc = Config(copy.deepcopy(PPO_DEFAULT_SESSION_CONFIG.to_dict()))
        sc.folder = tempfile.mkdtemp()
        ec.obs_spec = {'low_dim': {'flat_inputs': (c['D'],)}}
        ec.action_spec = {'dim': (c['A'],), 'type': 'continuous'}
        assert lc.algo.rnn.if_rnn_policy and lc.algo.ppo_mode == 'adapt'
    else:
        lc, ec, sc = ppo_configs(D=c['D'], A=c['A'], actor_h=c['actor_h'], critic_h=c['critic_h'], n_step=c['n'],
                                 stride=c['n'], B=c['B'], mode='clip' if c['mode'] == 'clip' else 'adapt')
        lc.algo.rnn.if_rnn_policy = True
        lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = c['horizon'], c['H'], 1
    lc.algo.consts.epoch_policy = epoch_policy
    lc.algo.consts.epoch_baseline = 1
    if lr is not None:
        lc.algo.network.lr_actor = lc.algo.network.lr_critic = lr
    return lc, ec, sc


def _layers(dims, gen):
    out = []
    for i in range(len(dims) - 1):
        b = 1.0 / np.sqrt(dims[i])
        out.append(((torch.rand(dims[i + 1], dims[i], generator=gen) * 2 - 1) * b, (torch.rand(dims[i + 1], generator=gen) * 2 - 1) * b))
    return out


def _stem_of(stem, buf):
    """(W_ih, W_hh, b_ih, b_hh) in torch's layout out of a flat stem-sized buffer (parameters or gradient)."""
    wi, bi = stem.ih.get_layer(0, buf[:stem.ih.size])
    wh, bh = stem.hh.get_layer(0, buf[stem.ih.size:])
    return wi, wh, bi, bh


def _rel(got, exp):
    return float((got.double() - exp).norm()) / max(float(exp.norm()), 1e-30)


def _maxrel(got, exp):
    return float((got.double() - exp).abs().max()) / max(float(exp.abs().max()), 1e-30)


def _check(pairs, what, bar=RNN_LEARN_BAR):
    worst = 0.0
    for got, exp, nm in pairs:
        exp = exp.to(got.device)
        r, m = _rel(got, exp), _maxrel(got, exp)
        worst = max(worst, r, m)
        assert r <= bar and m <= bar, (what, nm, r, m)
    print('measured', what, worst)
    return worst


def _check_joint(net, stem, g, ref, what, extra=None):
    """g = [head | stem] gradient buffer against a grad_ref result (``grads``, ``stem``, ``g_log_var``)."""
    pairs = []
    for l, (rw, rb) in enumerate(ref['grads']):
        gw, gb = net.get_layer(l, buf=g[:net.size])
        pairs += [(gw, rw, 'W%d' % l), (gb, rb, 'b%d' % l)]
    if extra is not None:
        pairs.append((net.extra_view(g[:net.size]), extra, 'log_var'))
    pairs += [(t, e, nm) for t, e, nm in zip(_stem_of(stem, g[net.size:]), ref['stem'], ['W_ih', 'W_hh', 'b_ih', 'b_hh'])]
    return _check(pairs, what)


def _joint_norm(ref, extra=None):
    s = sum(float(t.pow(2).sum()) for wb in ref['grads'] for t in wb) + sum(float(t.pow(2).sum()) for t in ref['stem'])
    if extra is not None:
        s += float(extra.pow(2).sum())
    return math.sqrt(s)


def _setup(c, monkeypatch, epoch_policy=1, lr=None, seed=0, graph=False):
    """A learner with random head / stem / z-filter parameters and a batch whose first eff_len steps have no head unit
    within 2e-5 of a relu kink under the float64 LSTM features (rows redrawn, as _clear_relu_ties does)."""
    from surreal_b200.learner import PPOLearner
    monkeypatch.setenv('SB200_CUDA_GRAPH', '1' if graph else '0')
    lc, ec, sc = _configs(c, epoch_policy, lr)
    B, n, A, D = lc.replay.batch_size, lc.algo.n_step, c['A'], c['D']
    Hh, hz = lc.algo.rnn.rnn_hidden, lc.algo.rnn.horizon
    E = n - hz + 1
    mode = c.get('mode', 'adapt')
    gen = torch.Generator().manual_seed(B + n + Hh + seed)
    ah, ch = list(lc.model.actor_fc_hidden_sizes), list(lc.model.critic_fc_hidden_sizes)
    al, cl = _layers([Hh] + ah + [A], gen), _layers([Hh] + ch + [1], gen)
    k = 1.0 / math.sqrt(Hh)
    u = lambda *s: (torch.rand(*s, generator=gen) * 2 - 1) * k  # noqa: E731
    stem = (u(4 * Hh, D), u(4 * Hh, Hh), u(4 * Hh), u(4 * Hh))
    log_var = torch.zeros(1, A) - 1.0
    zs = torch.cat([torch.randn(D, generator=gen) * 50, 500 * (1.5 + torch.rand(D, generator=gen)), torch.tensor([500.0])])
    obs = torch.randn(B, n, D, generator=gen) * 1.2
    obs_next = torch.randn(B, 1, D, generator=gen) * 1.2
    h0, c0 = torch.randn(B, Hh, generator=gen) * 0.3, torch.randn(B, Hh, generator=gen) * 0.5
    stem_d, zs_d = [t.to(DEV) for t in stem], zs.to(DEV)
    for _ in range(50):
        feat = R.rnn_features(stem_d, obs[:, :E].to(DEV), h0.to(DEV), c0.to(DEV), zs_d)
        bad = ((R.hidden_margin(feat, al) < 2e-5) | (R.hidden_margin(feat, cl) < 2e-5)).cpu().view(B, E)
        if not bool(bad.any()):
            break
        obs[:, :E][bad] = torch.randn(int(bad.sum()), D, generator=gen) * 1.2
    assert not bool(bad.any()), 'could not clear relu ties'
    with torch.no_grad():
        feat = R.rnn_features(stem_d, obs.to(DEV), h0.to(DEV), c0.to(DEV), zs_d)
        mu = torch.tanh(R.trunk(feat, [(R.f64(w).to(DEV), R.f64(b).to(DEV)) for w, b in al])).cpu()
    pd = torch.cat([mu, torch.exp(R.f64(log_var)).expand(B * n, A)], 1).float().view(B, n, 2 * A).numpy()
    rng = np.random.default_rng(B + n + seed)
    pd[:, :, A:] *= np.exp(rng.uniform(-0.25, 0.25, (B, 1, 1))).astype(np.float32)
    actions = np.clip(rng.standard_normal((B, n, A)) * pd[:, :, A:] + pd[:, :, :A], -1, 1).astype(np.float32)
    rewards = (rng.standard_normal((B, n)) * 0.3).astype(np.float32)
    dones = (rng.random((B, n)) < 0.02).astype(np.float32)
    L = PPOLearner(lc, ec, sc)
    assert L.rnn and L.eff_len == E and not L.use_epoch_kernel
    L.model.actor.load_layers(al, extra=log_var)
    L.model.critic.load_layers(cl)
    L.model.rnn_stem.load_torch(dict(zip(['weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0'], stem)))
    L.model.z_stats.copy_(zs_d)
    L.ref_target_model.update_target_params(L.model)
    ref_layers = al
    if mode != 'clip':
        # a reference policy away from the learner's: beta KL has a gradient of its own, and with 'adapt-hinge' the
        # pre-step KL is above 2 kl_target (the hinge is active)
        shift = 0.08 if mode == 'adapt-hinge' else 0.02
        ref_layers = al[:-1] + [(al[-1][0], al[-1][1] + shift * torch.sign(torch.randn(A, generator=gen)))]
        L.ref_target_model.actor.load_layers(ref_layers, extra=log_var)
    batch = {'obs': obs.numpy(), 'obs_next': obs_next.numpy(), 'actions': actions, 'rewards': rewards, 'dones': dones,
             'persistent_infos': [pd], 'onetime_infos': [h0[:, None].numpy(), c0[:, None].numpy()]}
    data = dict(obs=obs, obs_next=obs_next, h0=h0, c0=c0, pd=torch.from_numpy(pd), actions=torch.from_numpy(actions),
                rewards=torch.from_numpy(rewards), dones=torch.from_numpy(dones), ref_layers=ref_layers, log_var=log_var,
                zs=zs, E=E, mode=mode, stem=stem, al=al, cl=cl)
    return L, batch, data


def _record(L):
    """Wrap the epochs: per policy / value epoch, the parameters it starts from, the relu masks its backward used and
    the [head | stem] gradient it stepped."""
    rec = {'policy': [], 'value': []}
    for kind, tr, head in (('policy', L.actor_optim, L.model.actor), ('value', L.critic_optim, L.model.critic)):
        back = tr.backward

        def backward(*a, _tr=tr, _back=back, _kind=kind, **k):
            rec[_kind][-1]['masks'] = [(h[:, :n] > 0).clone() for h, n in zip(_tr.h[:-1], _tr.net.dims[1:-1])]
            return _back(*a, **k)
        tr.backward = backward
    pol, val = L._policy_epoch, L._value_epoch

    def policy_epoch(*a, **k):
        rec['policy'].append({'head': L.model.actor.params.clone(), 'stem': L.model.rnn_stem.params.clone()})
        pol(*a, **k)
        rec['policy'][-1].update(grad=L._g_actor.clone(), stem_after=L.model.rnn_stem.params.clone())

    def value_epoch(*a, **k):
        rec['value'].append({'head': L.model.critic.params.clone(), 'stem': L.model.rnn_stem.params.clone()})
        val(*a, **k)
        rec['value'][-1].update(grad=L._g_critic.clone())
    L._policy_epoch, L._value_epoch = policy_epoch, value_epoch
    return rec


def _ref_pd(L, d):
    """The reference policy on the update rows, in float64 (the reference model's stem = the learner's before learn())."""
    E, A = d['E'], L.action_dim
    with torch.no_grad():
        feat = R.rnn_features([t.to(DEV) for t in d['stem']], d['obs'][:, :E].to(DEV), d['h0'].to(DEV), d['c0'].to(DEV),
                              d['zs'].to(DEV))
        mean = torch.tanh(R.trunk(feat, [(R.f64(w).to(DEV), R.f64(b).to(DEV)) for w, b in d['ref_layers']]))
    return torch.cat([mean, torch.exp(R.f64(d['log_var'])).to(DEV).expand(mean.shape[0], A)], 1)


def _policy_ref(L, d, snap, ref_pd, masks=None):
    E, A = d['E'], L.action_dim
    net, stem = L.model.actor, L.model.rnn_stem
    layers = [net.get_layer(l, buf=snap['head']) for l in range(net.n_layers)]
    log_var = net.extra_view(snap['head'])
    args = (_stem_of(stem, snap['stem']), layers, log_var, d['obs'][:, :E].to(DEV), d['h0'].to(DEV), d['c0'].to(DEV),
            d['actions'][:, :E].to(DEV), L._adv, d['pd'][:, :E].to(DEV))
    if d['mode'] == 'clip':
        return R.ppo_policy_rnn(*args, 'clip', zs=d['zs'].to(DEV), masks=masks, clip_eps=L.clip_epsilon)
    r = R.ppo_policy_rnn(*args, 'adapt', zs=d['zs'].to(DEV), masks=masks, ref=ref_pd, beta=L.beta, kl_target=L.kl_target,
                         eta=L.eta)
    return r


def _value_ref(L, d, snap, masks=None):
    E, net = d['E'], L.model.critic
    layers = [net.get_layer(l, buf=snap['head']) for l in range(net.n_layers)]
    return R.value_rnn(_stem_of(L.model.rnn_stem, snap['stem']), layers, d['obs'][:, :E].to(DEV), d['h0'].to(DEV),
                       d['c0'].to(DEV), L._ret, zs=d['zs'].to(DEV), masks=masks)


def _gae64(rewards, values, dones, gamma, lam, hz, norm):
    """Horizon-windowed GAE and returns (ppo.py:389-406) in float64."""
    v = values.clone()
    v[:, 1:] *= 1 - dones
    tds = rewards + gamma * v[:, 1:] - v[:, :-1]
    n = rewards.shape[1]
    E = n - hz + 1
    g = gamma ** torch.arange(hz, dtype=torch.float64, device=v.device)
    gl = g * lam ** torch.arange(hz, dtype=torch.float64, device=v.device)
    ret = torch.stack([(g * rewards[:, s:s + hz]).sum(1) + v[:, s + hz] * gamma ** hz for s in range(E)], 1)
    adv = torch.stack([(tds[:, s:s + hz] * gl).sum(1) for s in range(E)], 1)
    if norm:
        adv = (adv - adv.mean()) / max(float(adv.std()), 1e-4)
    return adv, ret


@pytest.mark.parametrize('case', list(CASES))
def test_rnn_learn_gradients(case, monkeypatch):
    """One policy and one value epoch: [head | stem] gradients of both optimisers, the gradient norms, the stem's Adam
    moments of each optimiser, the critic pass, the horizon GAE and the z-filter update."""
    c = CASES[case]
    L, batch, d = _setup(c, monkeypatch)
    rec = _record(L)
    z_before = L.model.z_stats.clone()
    st = L.learn(batch)
    torch.cuda.synchronize()
    B, n, E, A = L.batch_size, L.n_step, d['E'], L.action_dim
    assert len(rec['policy']) == 1 and len(rec['value']) == 1
    assert torch.equal(z_before, d['zs'].to(DEV))
    # critic pass over all B (n + 1) rows from the window's initial cells, then float64 GAE on float64 values
    with torch.no_grad():
        full = torch.cat([d['obs'], d['obs_next']], 1).to(DEV)
        feat = R.rnn_features([t.to(DEV) for t in d['stem']], full, d['h0'].to(DEV), d['c0'].to(DEV), d['zs'].to(DEV))
        v64 = R.trunk(feat, [(R.f64(w).to(DEV), R.f64(b).to(DEV)) for w, b in d['cl']]).view(B, n + 1)
    ev = _maxrel(L._values.view(B, n + 1), v64)
    print('measured values', case, ev)
    assert ev <= VALUE_BAR, ev
    adv64, ret64 = _gae64(R.f64(d['rewards']).to(DEV), v64, R.f64(d['dones']).to(DEV), L.gamma, L.lam, L.horizon, L.norm_adv)
    ea = float((L._adv.double() - adv64).abs().max())
    er = float((L._ret.double() - ret64).abs().max()) / max(1.0, float(ret64.pow(2).mean().sqrt()))
    print('measured gae', case, ea, er)
    assert L._adv.shape == (B, E) and ea <= GAE_BAR and er <= GAE_BAR, (ea, er)
    # the policy epoch: gradients at the parameters before learn()
    ref_pd = _ref_pd(L, d) if d['mode'] != 'clip' else None
    rp = _policy_ref(L, d, rec['policy'][0], ref_pd)
    if d['mode'] != 'clip':
        assert rp['hinge'] == (d['mode'] == 'adapt-hinge')
        assert abs(float(rp['kl']) - 2 * L.kl_target) > 1e-3 * 2 * L.kl_target and float(rp['kl']) > 1e-3
    ga = rec['policy'][0]['grad']
    _check_joint(L.model.actor, L.model.rnn_stem, ga, rp, 'actor ' + case, extra=rp['g_log_var'])
    # the value epoch runs on the stem the actor has just stepped
    sv = rec['value'][0]['stem']
    assert torch.equal(sv, rec['policy'][0]['stem_after']) and not torch.equal(sv, rec['policy'][0]['stem'])
    rv = _value_ref(L, d, rec['value'][0], masks=rec['value'][0]['masks'])
    gc = rec['value'][0]['grad']
    _check_joint(L.model.critic, L.model.rnn_stem, gc, rv, 'critic ' + case)
    assert torch.equal(L._g_actor, ga) and torch.equal(L._g_critic, gc)
    # the clipped norm is the JOINT norm of head (+ log_var) and stem
    na, nc = _joint_norm(rp, rp['g_log_var']), _joint_norm(rv)
    ra, rc = abs(st['grad_norm_actor'] - na) / na, abs(st['grad_norm_critic'] - nc) / nc
    print('measured gradnorm', case, ra, rc)
    assert ra <= GN_BAR and rc <= GN_BAR, (st['grad_norm_actor'], na, st['grad_norm_critic'], nc)
    # each optimiser keeps its own Adam state for the shared stem: after one step m = (1 - b1) g', v = (1 - b2) g'^2 with
    # g' its OWN clipped stem gradient
    ns = L.model.actor.size
    for tr, g, nrm, nm in ((L.actor_rnn, ga[ns:], st['grad_norm_actor'], 'actor'),
                           (L.critic_rnn, gc[L.model.critic.size:], st['grad_norm_critic'], 'critic')):
        gcl = g.double() * min(1.0, 5.0 / (nrm + 1e-6))
        em, ev2 = _rel(tr.exp_avg, 0.1 * gcl), _rel(tr.exp_avg_sq, 0.001 * gcl * gcl)
        print('measured moments', case, nm, em, ev2)
        assert em <= MOMENT_BAR and ev2 <= MOMENT_BAR, (nm, em, ev2)
    # the z-filter counts the B * eff_len rows the updates trained on, after the updates
    x = R.f64(d['obs'][:, :E]).reshape(B * E, -1).to(DEV)
    D = x.shape[1]
    z = L.model.z_stats.double()
    assert float(z[2 * D]) == float(z_before[2 * D]) + B * E
    exp = torch.cat([z_before[:2 * D].double() + torch.cat([x.sum(0), (x * x).sum(0)])])
    ez = float((z[:2 * D] - exp).abs().max()) / float(exp.abs().max())
    print('measured zfilter', case, ez)
    assert ez <= ZF_BAR, ez


def test_rnn_policy_epochs_reuse_saved_activations(monkeypatch):
    """Three policy epochs of the default config: every epoch's gradient matches float64 at the parameters THAT epoch
    starts from.  Epochs 2 and 3 train on the activations the previous epoch's post-step forward saved (fresh=False),
    so a stale gate, cell or h_prev buffer shows up here."""
    c = CASES['default']
    L, batch, d = _setup(c, monkeypatch, epoch_policy=3, lr=3e-4, seed=1)
    rec = _record(L)
    L.learn(batch)
    torch.cuda.synchronize()
    assert L.last_n_policy_epochs == 3 and len(rec['policy']) == 3
    ref_pd = _ref_pd(L, d)
    for e, snap in enumerate(rec['policy']):
        if e > 0:
            assert torch.equal(snap['stem'], rec['policy'][e - 1]['stem_after'])
            assert not torch.equal(snap['stem'], rec['policy'][e - 1]['stem'])
        # epoch 0 runs on the tie-free parameters; later epochs take the relu decisions from the kernel's own activations
        rp = _policy_ref(L, d, snap, ref_pd, masks=snap['masks'] if e > 0 else None)
        _check_joint(L.model.actor, L.model.rnn_stem, snap['grad'], rp, 'actor epoch %d' % e, extra=rp['g_log_var'])
    rv = _value_ref(L, d, rec['value'][0], masks=rec['value'][0]['masks'])
    assert torch.equal(rec['value'][0]['stem'], rec['policy'][-1]['stem_after'])
    _check_joint(L.model.critic, L.model.rnn_stem, rec['value'][0]['grad'], rv, 'critic after 3 policy epochs')


@pytest.mark.parametrize('lr,stops', [(1e-4, False), (3e-2, True)])
def test_rnn_learn_graph_matches_eager(lr, stops, monkeypatch):
    """The default config with its 10 + 10 epochs: the captured learn() (KL early stop as a device flag) and the eager
    one (host break) leave bit-identical parameters, Adam states and z-filter, whether the early stop fires or not."""
    c = CASES['default']
    out = []
    for graph in (True, False):
        L, batch, _ = _setup(c, monkeypatch, epoch_policy=10, lr=lr, seed=2, graph=graph)
        L.learn(batch)
        torch.cuda.synchronize()
        assert L.use_cuda_graph == graph
        out.append((L.last_n_policy_epochs, [t.clone() for t in (
            L.model.actor.params, L.model.critic.params, L.model.rnn_stem.params, L.model.z_stats, L.actor_rnn.exp_avg,
            L.actor_rnn.exp_avg_sq, L.critic_rnn.exp_avg, L.critic_rnn.exp_avg_sq, L.actor_optim.exp_avg,
            L.critic_optim.exp_avg)]))
    assert out[0][0] == out[1][0]
    assert (out[0][0] < 10) == stops, out[0][0]
    for a, b in zip(out[0][1], out[1][1]):
        assert torch.equal(a, b)

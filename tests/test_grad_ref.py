"""The float64 gradient references of tests/grad_ref.py against the oracle's own float32 ``loss.backward()`` at small
shapes (CPU only).  This pins the semantics the kernels are held to: max(1)[0] sends the gradient to the first
maximum, clamp(min=1e-5) on the likelihood passes it where x >= min, adapt mode clamps the behaviour likelihood at
1e-2, the KL hinge applies only when the pre-step KL is above 2 kl_target, and std = exp(log_var)."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import grad_ref as R
from oracle import nets as onets
from oracle.ppo import OraclePPOLearner

D, H1, H2, A, B = 7, 12, 9, 3, 96


def _layers(dims, gen, scale=0.6):
    return [((torch.rand(dims[i + 1], dims[i], generator=gen) * 2 - 1) * scale,
             (torch.rand(dims[i + 1], generator=gen) * 2 - 1) * scale) for i in range(len(dims) - 1)]


def _close(got64, exp32, what, rtol=4e-6):
    """float32 autograd carries ~1e-7 relative rounding per operation: per tensor, the relative L2 difference
    measured worst 4.6e-7 over the MLP cases below and 8.9e-7 over the RNN-mode ones (LSTM stem); bar 4e-6."""
    g, e = got64.double(), exp32.double()
    err = float((g - e).norm()) / max(float(e.norm()), 1e-30)
    assert err <= rtol, (what, err)


def _policy_batch(gen, pert=0.35):
    """Rows in every regime: ratios across and outside the clip band with both signs of advantage, dead rows (the
    likelihood under the learner is < 1e-5) and behaviour likelihoods below 1e-2."""
    al = _layers([D, H1, H2, A], gen)
    log_var = torch.full((1, A), -0.8) + torch.rand(1, A, generator=gen) * 0.4
    obs = torch.randn(B, D, generator=gen)
    with torch.no_grad():
        mean = torch.tanh(onets.mlp_trunk(obs, al))
    bm = (mean + torch.randn(B, A, generator=gen) * pert).clamp(-0.95, 0.95)
    bs = torch.exp(log_var).expand(B, A) * torch.exp(torch.randn(B, 1, generator=gen) * 0.3)
    act = bm + torch.randn(B, A, generator=gen) * bs
    act[:6] = mean[:6] + 9.0 * torch.exp(log_var)                       # dead rows: learner likelihood < 1e-5
    adv = torch.randn(B, generator=gen)
    return al, log_var, obs, act, adv, torch.cat([bm, bs], 1)


def _oracle(al, log_var, cl, mode, **c):
    return OraclePPOLearner(al, log_var, cl or al, None, A, 1, B, ppo_mode=mode, **c)


def test_clip_loss_gradients_match_oracle():
    gen = torch.Generator().manual_seed(0)
    al, log_var, obs, act, adv, behave = _policy_batch(gen)
    O = _oracle(al, log_var, None, 'clip')
    loss, st = O._clip_loss(obs, act, adv, behave)
    loss.backward()
    r = R.ppo_policy(al, log_var, obs, act, adv, behave, 'clip', clip_eps=O.clip_epsilon)
    ratio = r['ratio']
    # the batch covers every branch of max(surr, clipped surr)
    assert bool(((ratio < 0.8) & (adv > 0)).any()) and bool(((ratio < 0.8) & (adv < 0)).any())
    assert bool(((ratio > 1.2) & (adv > 0)).any()) and bool(((ratio > 1.2) & (adv < 0)).any())
    assert bool(((ratio > 0.8) & (ratio < 1.2)).any())
    assert abs(float(r['loss']) - loss.item()) <= 1e-6 * max(1.0, abs(loss.item()))
    assert abs(float(r['surr']) - st['_surr_loss']) <= 1e-6 * max(1.0, abs(st['_surr_loss']))
    assert abs(float(r['entropy']) - st['_entropy']) <= 1e-6
    for l in range(3):
        _close(r['grads'][l][0], O.actor[l][0].grad, ('W', l))
        _close(r['grads'][l][1], O.actor[l][1].grad, ('b', l))
    _close(r['g_log_var'], O.log_var.grad.view(-1), 'log_var')
    # dead rows contribute nothing to the head gradient
    assert float(r['g_pre'][:6].abs().max()) == 0.0


@pytest.mark.parametrize('hinge', [False, True])
def test_adapt_loss_gradients_match_oracle(hinge):
    gen = torch.Generator().manual_seed(1)
    al, log_var, obs, act, adv, behave = _policy_batch(gen)
    ref_layers = [(w + torch.randn(w.shape, generator=gen) * 0.15, b) for w, b in al]
    with torch.no_grad():
        ref = onets.ppo_actor(obs, ref_layers, log_var - 0.1)
        klm = float(R.kl(R.f64(ref[:, :A]), R.f64(ref[:, A:]), torch.tanh(R.f64(onets.mlp_trunk(obs, al))),
                         torch.exp(R.f64(log_var)).expand(B, A)).mean())
    kl_target = klm / 2 * (0.7 if hinge else 1.4)                   # 30 % away from the hinge's branch point
    O = _oracle(al, log_var, None, 'adapt', kl_target=kl_target)
    loss, st = O._adapt_loss(obs, act, adv, behave, ref)
    loss.backward()
    r = R.ppo_policy(al, log_var, obs, act, adv, behave, 'adapt', ref=ref, beta=O.beta, kl_target=kl_target,
                     eta=O.c['kl_cutoff_coeff'])
    assert r['hinge'] == hinge
    lik_b = R.likelihood(R.f64(act), R.f64(behave[:, :A]), R.f64(behave[:, A:])).view(-1)
    assert bool((lik_b < 1e-2).any()) and bool((lik_b > 1e-2).any())
    assert abs(float(r['loss']) - loss.item()) <= 1e-6 * max(1.0, abs(loss.item()))
    assert abs(float(r['kl']) - st['_pol_kl']) <= 1e-6
    for l in range(3):
        _close(r['grads'][l][0], O.actor[l][0].grad, ('W', l))
        _close(r['grads'][l][1], O.actor[l][1].grad, ('b', l))
    _close(r['g_log_var'], O.log_var.grad.view(-1), 'log_var')


def test_value_loss_gradients_match_oracle():
    gen = torch.Generator().manual_seed(2)
    cl = _layers([D, H1, H2, 1], gen)
    obs, ret = torch.randn(B, D, generator=gen), torch.randn(B, generator=gen)
    O = _oracle(cl[:2] + [(torch.zeros(A, H2), torch.zeros(A))], torch.zeros(1, A), cl, 'clip')
    values = O.forward_critic(obs)                                    # _value_update's loss, without its step
    loss = (values - ret.view(-1, 1)).pow(2).mean()
    loss.backward()
    r = R.value(cl, obs, ret)
    assert abs(float(r['loss']) - loss.item()) <= 1e-6 * loss.item()
    ev = 1 - torch.var(ret.view(-1, 1) - values.detach()) / torch.var(ret.view(-1, 1))
    assert abs(float(r['explained_var']) - float(ev)) <= 1e-5
    for l in range(3):
        _close(r['grads'][l][0], O.critic[l][0].grad, ('W', l))
        _close(r['grads'][l][1], O.critic[l][1].grad, ('b', l))


def test_ddpg_losses_match_oracle():
    gen = torch.Generator().manual_seed(3)
    al = _layers([D, H1, H2, A], gen)
    cl = _layers([D, H1], gen) + _layers([H1 + A, H2, 1], gen)
    obs = torch.randn(B, D, generator=gen)
    act = torch.rand(B, A, generator=gen) * 2 - 1
    y = torch.randn(B, 1, generator=gen)
    c32 = [(w.clone().requires_grad_(True), b.clone().requires_grad_(True)) for w, b in cl]
    q = onets.ddpg_critic(obs, act, c32)
    nn.MSELoss()(q, y).backward()
    r = R.ddpg_critic(cl, obs, act, y)
    for l in range(3):
        _close(r['grads'][l][0], c32[l][0].grad, ('critic W', l))
        _close(r['grads'][l][1], c32[l][1].grad, ('critic b', l))
    assert abs(float(r['q_mean']) - float(q.mean())) <= 1e-6
    # importance weights: mean(w (q - y)^2); unit weights are the plain MSE
    w = torch.rand(B, generator=gen) + 0.1
    c32 = [(w_.clone().requires_grad_(True), b.clone().requires_grad_(True)) for w_, b in cl]
    (w.view(-1, 1) * (onets.ddpg_critic(obs, act, c32) - y) ** 2).mean().backward()
    rw = R.ddpg_critic(cl, obs, act, y, weights=w)
    r1 = R.ddpg_critic(cl, obs, act, y, weights=torch.ones(B))
    for l in range(3):
        _close(rw['grads'][l][0], c32[l][0].grad, ('weighted critic W', l))
        _close(rw['grads'][l][1], c32[l][1].grad, ('weighted critic b', l))
        assert torch.equal(r1['grads'][l][0], r['grads'][l][0]) and torch.equal(r1['grads'][l][1], r['grads'][l][1])
    a32 = [(w.clone().requires_grad_(True), b.clone().requires_grad_(True)) for w, b in al]
    (-onets.ddpg_critic(obs, onets.ddpg_actor(obs, a32), cl).mean()).backward()
    r = R.ddpg_actor(al, cl, obs)
    for l in range(3):
        _close(r['grads'][l][0], a32[l][0].grad, ('actor W', l))
        _close(r['grads'][l][1], a32[l][1].grad, ('actor b', l))
    # g_action is what grad_wrt_aux computes; through tanh it gives g_pre
    assert torch.allclose(r['g_pre'], r['g_action'] * (1 - torch.tanh(R.trunk(R.f64(obs), [(R.f64(w), R.f64(b)) for w, b in al])) ** 2),
                          rtol=1e-12)


@pytest.mark.parametrize('B,L,Din,H,cells', [(5, 1, 3, 4, True), (3, 9, 7, 6, False), (4, 6, 2, 1, True)])
def test_lstm_matches_torch_lstm(B, L, Din, H, cells):
    """grad_ref.lstm against torch.nn.LSTM(dtype=float64): outputs, final cells and the gradients of every weight and
    of the initial cells agree to float64 rounding."""
    gen = torch.Generator().manual_seed(B * 100 + L * 10 + H)
    ref = nn.LSTM(Din, H, 1, batch_first=True, dtype=torch.float64)
    with torch.no_grad():
        for p in ref.parameters():
            p.copy_(torch.rand(p.shape, generator=gen, dtype=torch.float64) * 1.6 - 0.8)
    x = torch.randn(B, L, Din, generator=gen, dtype=torch.float64)
    h0 = torch.randn(B, H, generator=gen, dtype=torch.float64).requires_grad_(True)
    c0 = torch.randn(B, H, generator=gen, dtype=torch.float64).requires_grad_(True)
    seed = torch.randn(B, L, H, generator=gen, dtype=torch.float64)
    out, (hn, cn) = ref(x, (h0[None], c0[None])) if cells else ref(x)
    ((out * seed).sum() + hn.sum() + 0.5 * cn.sum()).backward()
    w = [ref.weight_ih_l0, ref.weight_hh_l0, ref.bias_ih_l0, ref.bias_hh_l0]
    mine = [R.f64(t).requires_grad_(True) for t in w]
    h0m, c0m = R.f64(h0).requires_grad_(True), R.f64(c0).requires_grad_(True)
    r = R.lstm(x, h0m if cells else None, c0m if cells else None, *mine)
    loss = (r['h'] * seed).sum() + r['h_last'].sum() + 0.5 * r['c_last'].sum()
    gs = torch.autograd.grad(loss, mine + ([h0m, c0m] if cells else []))
    tol = 1e-12
    assert float((r['h'] - out).abs().max()) <= tol
    assert float((r['h_last'] - hn[0]).abs().max()) <= tol and float((r['c_last'] - cn[0]).abs().max()) <= tol
    assert torch.equal(r['h'][:, -1], r['h_last']) and torch.equal(r['c'][:, -1], r['c_last'])
    for g, p in zip(gs[:4], w):
        assert float((g - p.grad).abs().max()) <= tol * max(1.0, float(p.grad.abs().max()))
    if cells:
        assert float((gs[4] - h0.grad).abs().max()) <= tol and float((gs[5] - c0.grad).abs().max()) <= tol
    # the activated gates are what the pre-activations say
    G = torch.stack(r['pre'], 1)
    assert torch.allclose(r['gates'][..., :2 * H], torch.sigmoid(G[..., :2 * H]), rtol=0, atol=1e-15)
    assert torch.allclose(r['gates'][..., 2 * H:3 * H], torch.tanh(G[..., 2 * H:3 * H]), rtol=0, atol=1e-15)


RB, RL, RD, RH = 24, 5, 7, 6          # sequences, steps, observation width, LSTM width of the RNN-mode loss checks


def _rnn_policy_batch(gen, pert=0.35):
    """_policy_batch over B*L rows b*L + t of an LSTM stem: raw observations whose z-filter statistics put some
    columns at the eps floor of std and some rows past the +-5 clamp, and non-zero initial cells."""
    al = _layers([RH, H1, H2, A], gen)
    stem = [(torch.rand(4 * RH, RD, generator=gen) * 2 - 1) * 0.5, (torch.rand(4 * RH, RH, generator=gen) * 2 - 1) * 0.5,
            (torch.rand(4 * RH, generator=gen) * 2 - 1) * 0.3, (torch.rand(4 * RH, generator=gen) * 2 - 1) * 0.3]
    cnt = 40.0
    mean = torch.randn(RD, generator=gen)
    var = 0.5 + torch.rand(RD, generator=gen)
    mean[1], var[1] = 0.5, 0.0                     # std floored at eps; sums exact, so fp32 and fp64 agree on the floor
    zs = torch.cat([mean * cnt, (var + mean ** 2) * cnt, torch.tensor([cnt])])
    obs = mean + torch.randn(RB, RL, RD, generator=gen) * var.sqrt()
    obs[:, :, 1] = 0.5 + 1e-3 * torch.randint(-1, 2, (RB, RL), generator=gen)     # +-1e-3 / eps: clamped to +-5, or 0
    obs[::5, :, 3] += 9.0                                                 # past the +5 clamp
    h0, c0 = torch.randn(RB, RH, generator=gen) * 0.5, torch.randn(RB, RH, generator=gen) * 0.5
    log_var = torch.full((1, A), -0.8) + torch.rand(1, A, generator=gen) * 0.4
    feat = R.rnn_features(stem, obs, h0, c0, zs)
    with torch.no_grad():
        mu = torch.tanh(R.trunk(feat, [(R.f64(w), R.f64(b)) for w, b in al])).float()
    M = RB * RL
    bm = (mu + torch.randn(M, A, generator=gen) * pert).clamp(-0.95, 0.95)
    bs = torch.exp(log_var).expand(M, A) * torch.exp(torch.randn(M, 1, generator=gen) * 0.3)
    act = bm + torch.randn(M, A, generator=gen) * bs
    act[:6] = mu[:6] + 9.0 * torch.exp(log_var)                           # dead rows
    adv = torch.randn(RB, RL, generator=gen)
    return al, stem, log_var, zs, obs, h0, c0, act, adv, torch.cat([bm, bs], 1)


def _rnn_oracle(al, log_var, cl, stem, zs, mode, **c):
    from oracle.filters import ZFilter
    from oracle.ppo_rnn import OraclePPOLearnerRNN
    zf = ZFilter(RD).load(zs[:RD], zs[RD:2 * RD], zs[2 * RD:])
    st = dict(zip(['weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0'], stem))
    return OraclePPOLearnerRNN(al, log_var, cl, zf, st, A, RL, RB, 1, RH, 1, ppo_mode=mode, **c)


def _close_stem(r, O):
    for got, p, nm in zip(r['stem'], [O.rnn.weight_ih_l0, O.rnn.weight_hh_l0, O.rnn.bias_ih_l0, O.rnn.bias_hh_l0],
                          ['W_ih', 'W_hh', 'b_ih', 'b_hh']):
        _close(got, p.grad, nm)


@pytest.mark.parametrize('mode', ['clip', 'adapt', 'adapt-hinge'])
def test_rnn_policy_loss_gradients_match_oracle(mode):
    """ppo_policy_rnn against OraclePPOLearnerRNN's float32 loss.backward() through nn.LSTM: head, log_var and all four
    LSTM gradients; the initial cells are data (detached), the z-filter clamps and floors."""
    gen = torch.Generator().manual_seed(5 + len(mode))
    al, stem, log_var, zs, obs, h0, c0, act, adv, behave = _rnn_policy_batch(gen)
    if mode == 'clip':
        O = _rnn_oracle(al, log_var, al, stem, zs, 'clip')
        O.cells = (h0[None].clone(), c0[None].clone())
        loss, st = O._clip_loss(obs, act, adv.reshape(-1), behave)
        r = R.ppo_policy_rnn(stem, al, log_var, obs, h0, c0, act, adv, behave, 'clip', zs=zs, clip_eps=O.clip_epsilon)
        ratio = r['ratio']
        a = adv.reshape(-1)
        assert bool(((ratio < 0.8) & (a > 0)).any()) and bool(((ratio > 1.2) & (a < 0)).any())
        assert bool(((ratio > 0.8) & (ratio < 1.2)).any())
    else:
        ref_layers = [(w + torch.randn(w.shape, generator=gen) * 0.15, b) for w, b in al]
        with torch.no_grad():
            feat = R.rnn_features(stem, obs, h0, c0, zs)
            ref = torch.cat([torch.tanh(R.trunk(feat, [(R.f64(w), R.f64(b)) for w, b in ref_layers])),
                             torch.exp(R.f64(log_var) - 0.1).expand(RB * RL, A)], 1).float()
            mu = torch.tanh(R.trunk(feat, [(R.f64(w), R.f64(b)) for w, b in al]))
            klm = float(R.kl(R.f64(ref[:, :A]), R.f64(ref[:, A:]), mu, torch.exp(R.f64(log_var)).expand(RB * RL, A)).mean())
        kl_target = klm / 2 * (0.7 if mode == 'adapt-hinge' else 1.4)
        O = _rnn_oracle(al, log_var, al, stem, zs, 'adapt', kl_target=kl_target)
        O.cells = (h0[None].clone(), c0[None].clone())
        loss, st = O._adapt_loss(obs, act, adv.reshape(-1), behave, ref)
        r = R.ppo_policy_rnn(stem, al, log_var, obs, h0, c0, act, adv, behave, 'adapt', zs=zs, ref=ref, beta=O.beta,
                             kl_target=kl_target, eta=O.c['kl_cutoff_coeff'])
        assert r['hinge'] == (mode == 'adapt-hinge')
        assert abs(float(r['kl']) - st['_pol_kl']) <= 1e-6
    loss.backward()
    assert abs(float(r['loss']) - loss.item()) <= 1e-6 * max(1.0, abs(loss.item()))
    for l in range(3):
        _close(r['grads'][l][0], O.actor[l][0].grad, ('W', l))
        _close(r['grads'][l][1], O.actor[l][1].grad, ('b', l))
    _close(r['g_log_var'], O.log_var.grad.view(-1), 'log_var')
    _close_stem(r, O)
    if mode == 'clip':
        assert float(r['g_pre'][:6].abs().max()) == 0.0
    assert min(float(g.abs().max()) for g in r['stem']) > 0.0


def test_rnn_value_loss_gradients_match_oracle():
    gen = torch.Generator().manual_seed(8)
    al, stem, log_var, zs, obs, h0, c0, _, _, _ = _rnn_policy_batch(gen)
    cl = _layers([RH, H1, H2, 1], gen)
    ret = torch.randn(RB, RL, generator=gen)
    O = _rnn_oracle(al, log_var, cl, stem, zs, 'clip')
    O.cells = (h0[None].clone(), c0[None].clone())
    values = O.forward_critic(obs).squeeze(2)                        # _value_update's loss, without its step
    loss = (values - ret).pow(2).mean()
    loss.backward()
    r = R.value_rnn(stem, cl, obs, h0, c0, ret, zs=zs)
    assert abs(float(r['loss']) - loss.item()) <= 1e-6 * loss.item()
    for l in range(3):
        _close(r['grads'][l][0], O.critic[l][0].grad, ('W', l))
        _close(r['grads'][l][1], O.critic[l][1].grad, ('b', l))
    _close_stem(r, O)


def test_likelihood_clamp_passes_gradient_at_the_floor():
    """torch.clamp(min) passes the gradient where x >= min (so also at x == min): the kernels' live-row test."""
    x = torch.tensor([1e-5 * 0.5, 1e-5, 2e-5], dtype=torch.float64, requires_grad=True)
    torch.clamp(x, min=1e-5).sum().backward()
    assert x.grad.tolist() == [0.0, 1.0, 1.0]
    # max(1)[0] of a tie routes the gradient to the first column
    t = torch.tensor([[1.0, 1.0]], requires_grad=True)
    t.max(1)[0].sum().backward()
    assert t.grad.tolist() == [[1.0, 0.0]]
    assert np.isfinite(float(R.zfilter(torch.zeros(1, 2), torch.tensor([0.0, 0.0, 1e-5, 1e-5, 1e-5]))[0, 0]))

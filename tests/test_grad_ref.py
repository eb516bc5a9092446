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
    measured worst 4.6e-7 over the cases below; bar 4e-6."""
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
    a32 = [(w.clone().requires_grad_(True), b.clone().requires_grad_(True)) for w, b in al]
    (-onets.ddpg_critic(obs, onets.ddpg_actor(obs, a32), cl).mean()).backward()
    r = R.ddpg_actor(al, cl, obs)
    for l in range(3):
        _close(r['grads'][l][0], a32[l][0].grad, ('actor W', l))
        _close(r['grads'][l][1], a32[l][1].grad, ('actor b', l))
    # g_action is what grad_wrt_aux computes; through tanh it gives g_pre
    assert torch.allclose(r['g_pre'], r['g_action'] * (1 - torch.tanh(R.trunk(R.f64(obs), [(R.f64(w), R.f64(b)) for w, b in al])) ** 2),
                          rtol=1e-12)


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

"""The categorical PPO policy on the CPU: its float64 semantics (tests/cat_ref.py) against torch.distributions.Categorical
and autograd in float64, the clip / adapt losses and their logit gradients, the aggregator's one-hot encoding, the
configuration errors, and the sm_90a cross-compile of the kernels (csrc/ppo_cat.cu)."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import cat_ref as PD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_MAX = 4096                     # SB200_PPO_CAT_MAX_K
KS = [2, 3, 18, K_MAX]


def _logits(rows, K, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(rows, K, generator=g, dtype=torch.float64) * scale


def _one_hot(idx, K):
    return torch.nn.functional.one_hot(torch.as_tensor(idx), K).to(torch.float64)


@pytest.mark.parametrize('K', KS)
@pytest.mark.parametrize('saturate', [False, True])
def test_distribution_functions_match_torch_categorical(K, saturate):
    rows = 5
    lg = _logits(rows, K, K)
    if saturate:                 # softmax saturates: p underflows to 0 for most entries, the 1e-5 clamp binds
        lg = torch.where(lg > 0, torch.full_like(lg, 80.0), torch.full_like(lg, -80.0))
        lg[:, 0] = 80.0
        lg[:, 1] = -80.0
    ref = torch.distributions.Categorical(logits=lg)
    prob = PD.cat_prob(lg)
    assert prob.shape == (rows, 2 * K)
    assert torch.allclose(prob[:, :K], ref.probs, rtol=1e-12, atol=1e-300)
    assert torch.allclose(prob[:, K:], ref.logits, rtol=1e-12, atol=1e-12)
    a_idx = torch.arange(rows) % K
    if saturate:
        a_idx[:] = 1             # p_a = exp(-160) / ...: below the clamp
    a = _one_hot(a_idx, K)
    ll = PD.cat_loglikelihood(a, prob, K).view(-1)
    assert torch.allclose(ll, ref.log_prob(a_idx), rtol=1e-12, atol=1e-12)
    lik = PD.cat_likelihood(a, prob, K).view(-1)
    assert torch.allclose(lik, torch.clamp(ref.log_prob(a_idx).exp(), min=1e-5), rtol=1e-12, atol=0)
    ent = PD.cat_entropy(prob, K)
    assert torch.allclose(ent, ref.entropy(), rtol=1e-10, atol=1e-12)
    lg1 = _logits(rows, K, K + 1)
    prob1 = PD.cat_prob(lg1)
    kl = PD.cat_kl(prob, prob1, K)
    kl_ref = torch.distributions.kl_divergence(ref, torch.distributions.Categorical(logits=lg1))
    assert torch.allclose(kl, kl_ref, rtol=1e-10, atol=1e-10)
    assert torch.allclose(PD.cat_kl(prob, prob, K), torch.zeros(rows, dtype=torch.float64), atol=1e-12)


def test_likelihood_clamp_has_zero_gradient_where_it_binds():
    K = 3
    lg = torch.tensor([[80.0, -80.0, 0.0], [0.1, 0.2, 0.3]], dtype=torch.float64, requires_grad=True)
    a = _one_hot([1, 1], K)
    PD.cat_likelihood(a, PD.cat_prob(lg), K).sum().backward()
    assert float(lg.grad[0].abs().max()) == 0.0            # p_a ~ e^-160 < 1e-5
    p = torch.softmax(lg.detach()[1], 0)
    expect = p[1] * (torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64) - p)
    assert torch.allclose(lg.grad[1], expect, rtol=1e-12)


def test_maxprob_takes_the_lowest_index_among_ties():
    K = 18
    lg = torch.zeros(3, K, dtype=torch.float64)
    lg[0, [4, 9]] = 2.0
    lg[1, :] = -1.0
    lg[2, [17, 3, 11]] = 5.0
    got = PD.cat_maxprob(PD.cat_prob(lg).numpy(), K)
    assert got.tolist() == [4, 0, 3]


@pytest.mark.parametrize('K', [2, 3, 18])
def test_inverse_cdf_sampling(K):
    prob = PD.cat_prob(_logits(4, K, 7)).numpy()
    c = np.cumsum(prob[:, :K], axis=1)
    u = np.stack([np.zeros(4), c[:, 0] * 0.5, c[:, K // 2], np.full(4, 1.0)], axis=1)
    for col in range(u.shape[1]):
        got = PD.cat_sample(prob, K, u[:, col])
        for r in range(4):
            hits = np.nonzero(u[r, col] < c[r])[0]
            assert got[r] == (hits[0] if len(hits) else K - 1)
    assert (PD.cat_sample(prob, K, np.zeros(4)) == 0).all()


def test_philox_uniform_is_exact_and_in_range():
    from cat_ref import agent_uniform
    from oracle.philox import philox4x32_10
    u = agent_uniform(12345, 7, np.arange(1000))
    assert u.min() >= 0.0 and u.max() < 1.0
    x, _, _, _ = philox4x32_10(np.uint64(12345), np.uint64(7), np.arange(1000, dtype=np.uint64) << np.uint64(16))
    assert np.array_equal(u * 2.0 ** 24, (x >> np.uint32(8)).astype(np.float64))
    assert np.array_equal(u.astype(np.float32).astype(np.float64), u)            # exact in fp32


# -- losses ----------------------------------------------------------------------------------------------------------
def _loss_ref(mode, lg, a_idx, adv, behave_lg, ref_lg, eps, beta, eta, kl_target):
    """The reference's clip / adapt formulas (ppo.py:194-225, 250-285) written on torch.distributions.Categorical."""
    learn = torch.distributions.Categorical(logits=lg)
    lp = torch.clamp(learn.log_prob(a_idx).exp(), min=1e-5).view(-1, 1)
    bp = torch.clamp(torch.distributions.Categorical(logits=behave_lg).log_prob(a_idx).exp(), min=1e-5).view(-1, 1)
    if mode == 'clip':
        ratio = lp / bp
        surr = -ratio * adv.view(-1, 1)
        csurr = -torch.clamp(ratio, 1 - eps, 1 + eps) * adv.view(-1, 1)
        return torch.cat([surr, csurr], 1).max(1)[0].mean()
    kl = torch.distributions.kl_divergence(torch.distributions.Categorical(logits=ref_lg), learn).mean()
    loss = -(adv.view(-1, 1) * (lp / torch.clamp(bp, min=1e-2))).mean() + beta * kl
    if kl.item() - 2.0 * kl_target > 0:
        loss = loss + eta * (kl - 2.0 * kl_target).pow(2)
    return loss


def _oracle_learner(mode, K, D=5, kl_target=0.015, clip_epsilon=0.2, beta=1.0):
    from cat_ref import CatOraclePPOLearner
    g = torch.Generator().manual_seed(K)
    al = [(torch.randn(7, D, generator=g, dtype=torch.float64) * 0.4, torch.randn(7, generator=g, dtype=torch.float64) * 0.1),
          (torch.randn(K, 7, generator=g, dtype=torch.float64) * 0.4, torch.randn(K, generator=g, dtype=torch.float64) * 0.1)]
    cl = [(torch.randn(1, D, generator=g, dtype=torch.float64), torch.zeros(1, dtype=torch.float64))]
    O = CatOraclePPOLearner(al, cl, None, K, 1, 8, ppo_mode=mode, kl_target=kl_target, clip_epsilon_init=clip_epsilon,
                            beta_init=beta)
    return O, g


@pytest.mark.parametrize('K', KS)
@pytest.mark.parametrize('mode', ['clip', 'adapt_below', 'adapt_above'])
def test_oracle_losses_and_gradients_match_autograd_on_torch_categorical(K, mode):
    """The oracle learner's categorical clip / adapt loss and its gradient w.r.t. the actor parameters against the same
    formulas on torch.distributions.Categorical; the adapt eta penalty on both sides of 2 * kl_target."""
    ppo_mode = 'clip' if mode == 'clip' else 'adapt'
    kl_target = {'clip': 0.015, 'adapt_below': 1e3, 'adapt_above': 1e-6}[mode]
    O, g = _oracle_learner(ppo_mode, K, kl_target=kl_target)
    B, D = 8, 5
    obs = torch.randn(B, D, generator=g, dtype=torch.float64)
    a_idx = torch.randint(0, K, (B,), generator=g)
    a = _one_hot(a_idx, K)
    adv = torch.randn(B, generator=g, dtype=torch.float64)
    with torch.no_grad():
        from oracle import nets
        lg0 = nets.mlp_trunk(obs, O.actor)
        behave_lg = lg0 + torch.randn(B, K, generator=g, dtype=torch.float64) * 0.3
        ref_lg = lg0 + torch.randn(B, K, generator=g, dtype=torch.float64) * 0.5
    behave_pol, ref_pol = PD.cat_prob(behave_lg), PD.cat_prob(ref_lg)
    if ppo_mode == 'clip':
        loss, _ = O._clip_loss(obs, a, adv, behave_pol)
    else:
        loss, st = O._adapt_loss(obs, a, adv, behave_pol, ref_pol)
        above = st['_pol_kl'] - 2.0 * kl_target > 0
        assert above == (mode == 'adapt_above')
    grads = torch.autograd.grad(loss, O.actor_params)
    params = [p.detach().clone().requires_grad_(True) for p in O.actor_params]
    lg = nets.mlp_trunk(obs, [(params[0], params[1]), (params[2], params[3])])
    ref = _loss_ref(ppo_mode, lg, a_idx, adv, behave_lg, ref_lg, O.c['clip_epsilon_init'], O.c['beta_init'],
                    O.c['kl_cutoff_coeff'], kl_target)
    ref_grads = torch.autograd.grad(ref, params)
    assert abs(loss.item() - ref.item()) <= 1e-12 * max(1.0, abs(ref.item()))
    for gg, rg in zip(grads, ref_grads):
        assert torch.allclose(gg, rg, rtol=1e-9, atol=1e-14)


def test_oracle_categorical_learn_runs_and_omits_log_sig():
    O, g = _oracle_learner('adapt', 4)
    B, n, D, K = 8, 1, 5, 4
    obs = torch.randn(B, n, D, generator=g, dtype=torch.float64)
    with torch.no_grad():
        from oracle import nets
        pd0 = PD.cat_prob(nets.mlp_trunk(obs[:, 0], O.actor)).numpy()
    idx = PD.cat_sample(pd0, K, np.linspace(0.05, 0.95, B))
    batch = dict(obs=obs.numpy(), obs_next=torch.randn(B, 1, D, generator=g, dtype=torch.float64).numpy(),
                 actions=np.eye(K)[idx][:, None], rewards=np.linspace(-1, 1, B)[:, None], dones=np.zeros((B, n)),
                 pd=pd0[:, None])
    st = O.learn(batch)
    assert '_avg_log_sig' not in st and st['_entropy'] > 0 and O.n_policy_epochs[-1] >= 1


# -- aggregator ------------------------------------------------------------------------------------------------------
def test_aggregator_one_hot_encodes_discrete_actions():
    from surreal_b200.learner.aggregator import MultistepAggregatorWithInfo, SSARAggregator
    K, n = 5, 3
    spec = {'low_dim': {'flat_inputs': (2,)}}
    agg = MultistepAggregatorWithInfo(spec, {'type': 'discrete', 'dim': (K,)})
    rng = np.random.default_rng(0)
    idx = rng.integers(0, K, (4, n))
    exps = [{'obs': [{'low_dim': {'flat_inputs': np.zeros(2)}}] * n, 'obs_next': {'low_dim': {'flat_inputs': np.ones(2)}},
             'actions': list(idx[b]), 'rewards': [0.0] * n, 'dones': [0.0] * n, 'onetime_infos': [],
             'persistent_infos': [[np.zeros(2 * K, dtype=np.float32)] for _ in range(n)]} for b in range(4)]
    out = agg.aggregate(exps)
    assert out['actions'].dtype == np.float32 and out['actions'].shape == (4, n, K)
    assert np.array_equal(out['actions'].argmax(-1), idx) and np.array_equal(out['actions'].sum(-1), np.ones((4, n)))
    exps[0]['actions'][1] = K
    with pytest.raises(ValueError):
        agg.aggregate(exps)
    with pytest.raises(NotImplementedError):
        SSARAggregator(spec, {'type': 'discrete', 'dim': (K,)})


# -- configuration -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [1, K_MAX + 1])
def test_discrete_spec_outside_the_cap_is_a_config_error(K):
    from surreal_b200.model.ppo_net import make_pd
    from surreal_b200.session import ConfigError
    with pytest.raises(ConfigError):
        make_pd({'type': 'discrete', 'dim': (K,)})


def test_discrete_spec_selects_categorical_and_continuous_keeps_gaussian():
    from surreal_b200 import _lib
    from surreal_b200.model.ppo_net import make_pd, Categorical, DiagGauss
    assert isinstance(make_pd({'type': 'discrete', 'dim': (K_MAX,)}), Categorical)
    g = make_pd({'type': 'continuous', 'dim': (8,)})
    assert isinstance(g, DiagGauss) and g.pd_type == _lib.PD_GAUSSIAN == 0
    assert _lib.PPO_CAT_MAX_K == K_MAX


def test_data_parallel_refuses_a_categorical_policy():
    from surreal_b200.learner.ppo import PPOLearner
    with pytest.raises(NotImplementedError):
        PPOLearner.enable_data_parallel(types.SimpleNamespace(categorical=True, use_r_filter=False, rnn=False))


def test_header_cap_matches_binding():
    txt = open(os.path.join(ROOT, 'include', 'surreal_b200.h')).read()
    assert '#define SB200_PPO_CAT_MAX_K %d' % K_MAX in txt


def test_kernels_cross_compile_for_sm_90a(tmp_path):
    from surreal_b200 import build
    assert 'arch=compute_90a,code=sm_90a' in build.FLAGS
    if not os.path.exists(build.NVCC):
        pytest.skip('nvcc not installed')
    src = os.path.join(build.CSRC, 'ppo_cat.cu')
    r = subprocess.run([build.NVCC] + build.FLAGS + ['-c', src, '-o', str(tmp_path / 'ppo_cat.o')],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([sys.executable, '-m', 'surreal_b200.build'], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr

"""The categorical PPO policy on the GPU (csrc/ppo_cat.cu) against the float64 semantics of tests/cat_ref.py:
each kernel over its envelope, the sampler's Philox inverse CDF, the window staging of act() + DiscreteSyntheticEnv,
learn() in clip and adapt mode on the MLP, LSTM and CNN stems, graph replay against eager, and checkpoints."""
import copy

import numpy as np
import pytest
import torch

from helpers import ppo_configs
import cat_ref as PD
from cat_ref import agent_uniform

pytestmark = pytest.mark.gpu
DEV = 'cuda'
K_MAX = 4096
KS = [2, 3, 18, 64, K_MAX]
BS = [1, 32, 33, 256, 257, 4096]


def _lib():
    from surreal_b200 import _lib as L
    L.ensure_device()
    return L.lib()


def _p(t):
    return None if t is None else t.data_ptr()


def _close(got, exp, what):
    exp = np.asarray(exp, dtype=np.float64)
    got = np.asarray(got, dtype=np.float64)
    tol = 1e-5 * max(1.0, float(np.sqrt(np.mean(exp ** 2))) if exp.size else 1.0)
    err = float(np.abs(got - exp).max()) if exp.size else 0.0
    assert err <= tol, '%s: max err %.3e > %.3e' % (what, err, tol)


def _case(B, K, seed):
    """fp32 logits (some rows saturated at +-80, some with tied maxima), one-hot actions, advantages, behaviour / ref pd
    rows made by the oracle from perturbed logits."""
    rng = np.random.default_rng(seed)
    lg = (rng.standard_normal((B, K)) * 2.0).astype(np.float32)
    sat = rng.random(B) < 0.1
    lg[sat] = np.where(rng.random((int(sat.sum()), K)) < 0.5, 80.0, -80.0).astype(np.float32)
    tie = rng.random(B) < 0.1
    lg[tie, : min(K, 2)] = lg[tie].max(axis=1, keepdims=True) + 1.0
    a_idx = rng.integers(0, K, B)
    act = np.eye(K, dtype=np.float32)[a_idx]
    adv = rng.standard_normal(B).astype(np.float32)
    f64 = lambda x: torch.tensor(x, dtype=torch.float64)  # noqa: E731
    behave = PD.cat_prob(f64(lg + rng.standard_normal((B, K)) * 0.3)).numpy().astype(np.float32)
    ref = PD.cat_prob(f64(lg + rng.standard_normal((B, K)) * 0.3)).numpy().astype(np.float32)
    return lg, act, adv, behave, ref


def _dev(x):
    return torch.tensor(np.ascontiguousarray(x), device=DEV)


# -- 1. kernels against the float64 oracle -----------------------------------------------------------------------------
@pytest.mark.parametrize('K', KS)
@pytest.mark.parametrize('B', BS)
def test_make_pd_and_kl_and_final_stats(B, K):
    L = _lib()
    lg, act, adv, behave, ref = _case(B, K, 11 * B + K)
    d_lg, d_act, d_beh, d_ref = _dev(lg), _dev(act), _dev(behave), _dev(ref)
    pd = torch.zeros(B, 2 * K, device=DEV)
    assert L.sb200_ppo_cat_make_pd_f32(_p(d_lg), K, B, K, _p(pd), 2 * K, None) == 0
    exp = PD.cat_prob(torch.tensor(lg, dtype=torch.float64)).numpy()
    got = pd.cpu().numpy()
    _close(got[:, :K], exp[:, :K], 'p')
    _close(got[:, K:], exp[:, K:], 'log p')
    ws = torch.zeros(int(L.sb200_ppo_loss_workspace_bytes(B, K)), dtype=torch.uint8, device=DEV)
    stats = torch.zeros(32, device=DEV)
    stop = torch.zeros(1, dtype=torch.int32, device=DEV)
    kl_exp = float(PD.cat_kl(torch.tensor(ref, dtype=torch.float64), torch.tensor(exp), K).mean())
    # threshold above the KL: no stop; then below it: the flag is raised
    assert L.sb200_ppo_cat_kl_f32(_p(d_ref), 2 * K, _p(d_lg), K, B, K, _p(stats), 4, kl_exp * 2 + 1.0, _p(stop), _p(ws), None) == 0
    torch.cuda.synchronize()
    _close([float(stats[4])], [kl_exp], 'kl')
    assert int(stop) == 0 and float(stats[14]) == 1.0
    assert L.sb200_ppo_cat_kl_f32(_p(d_ref), 2 * K, _p(d_lg), K, B, K, _p(stats), 4, kl_exp * 0.5, _p(stop), _p(ws), None) == 0
    torch.cuda.synchronize()
    assert int(stop) == 1
    # a raised flag makes the KL kernel a no-op
    stop.fill_(1)
    stats.fill_(-7.0)
    assert L.sb200_ppo_cat_kl_f32(_p(d_ref), 2 * K, _p(d_lg), K, B, K, _p(stats), 4, 1.0, _p(stop), _p(ws), None) == 0
    torch.cuda.synchronize()
    assert bool((stats == -7.0).all())
    stats.zero_()
    assert L.sb200_ppo_cat_final_stats_f32(_p(d_lg), K, _p(d_act), K, _p(d_beh), 2 * K, _p(d_ref), 2 * K, B, K, _p(stats),
                                           _p(ws), None) == 0
    t64 = lambda x: torch.tensor(x, dtype=torch.float64)  # noqa: E731
    lb = PD.cat_likelihood(t64(act), t64(behave), K)
    lc = PD.cat_likelihood(t64(act), torch.tensor(exp), K)
    s = stats.cpu().numpy()
    _close([s[11], s[12], s[13]], [float(lb.mean()), float((lc / (lb + 1e-4)).mean()),
                                   float(PD.cat_kl(t64(ref), t64(behave), K).mean())], 'final stats')


@pytest.mark.parametrize('mode', ['clip', 'adapt_below', 'adapt_above'])
@pytest.mark.parametrize('K', KS)
@pytest.mark.parametrize('B', BS)
def test_policy_loss_and_logit_gradient(B, K, mode):
    L = _lib()
    lg, act, adv, behave, ref = _case(B, K, 7 * B + K)
    m = 0 if mode == 'clip' else 1
    eps, beta, eta = 0.2, 1.3, 250.0
    t64 = lambda x: torch.tensor(x, dtype=torch.float64)  # noqa: E731
    x = t64(lg).requires_grad_(True)
    learn = PD.cat_prob(x)
    lp, bp = PD.cat_likelihood(t64(act), learn, K), PD.cat_likelihood(t64(act), t64(behave), K)
    kl_mean = None
    if m == 0:
        ratio = lp / bp
        surr = -ratio * t64(adv).view(-1, 1)
        loss = torch.cat([surr, -torch.clamp(ratio, 1 - eps, 1 + eps) * t64(adv).view(-1, 1)], 1).max(1)[0].mean()
        kt = 0.015
    else:
        kl = PD.cat_kl(t64(ref), learn, K).mean()
        kl_mean = kl.item()
        kt = kl_mean * 10.0 if mode == 'adapt_below' else kl_mean / 10.0        # both sides of 2 * kl_target
        surr = -(t64(adv).view(-1, 1) * (lp / torch.clamp(bp, min=1e-2)))
        loss = surr.mean() + beta * kl
        if kl_mean - 2.0 * kt > 0:
            loss = loss + eta * (kl - 2.0 * kt).pow(2)
    loss.backward()
    ent = float(PD.cat_entropy(learn.detach(), K).mean())
    ldd = K + 5
    d_lg = _dev(lg)
    dlog = torch.full((B, ldd), 9.0, device=DEV)
    stats = torch.zeros(32, device=DEV)
    hyper = torch.tensor([eps, beta], dtype=torch.float64, device=DEV)
    ws = torch.zeros(int(L.sb200_ppo_loss_workspace_bytes(B, K)), dtype=torch.uint8, device=DEV)
    stop = torch.zeros(1, dtype=torch.int32, device=DEV)
    d_act, d_adv, d_beh, d_ref = _dev(act), _dev(adv), _dev(behave), _dev(ref)
    args = (m, _p(d_lg), K, _p(d_act), K, _p(d_adv), _p(d_beh), 2 * K, _p(d_ref), 2 * K, B, K, _p(hyper), eta, kt, _p(dlog),
            ldd, _p(stats), _p(ws), _p(stop), None)
    if m == 1:
        assert L.sb200_ppo_cat_kl_f32(_p(d_ref), 2 * K, _p(d_lg), K, B, K, _p(stats), 3, 0.0, _p(stop), _p(ws), None) == 0
    assert L.sb200_ppo_cat_policy_loss_f32(*args) == 0
    torch.cuda.synchronize()
    s = stats.cpu().numpy()
    _close([s[0]], [surr.mean().item()], 'surr')
    _close([s[1]], [loss.item()], 'loss')
    _close([s[2]], [ent], 'entropy')
    if m == 1:
        _close([s[3]], [kl_mean], 'kl_pre')
    g = dlog.cpu().numpy()
    _close(g[:, :K], x.grad.numpy(), 'dlogits')
    assert bool((dlog[:, K:] == 0).all())
    # stop flag set: a no-op
    stop.fill_(1)
    dlog.fill_(3.0)
    stats.fill_(3.0)
    assert L.sb200_ppo_cat_policy_loss_f32(*args) == 0
    torch.cuda.synchronize()
    assert bool((dlog == 3.0).all()) and bool((stats == 3.0).all())


# -- 2. sampler ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', KS)
@pytest.mark.parametrize('N', [1, 33, 1024, 4096])
def test_sampler_matches_the_philox_inverse_cdf(N, K):
    L = _lib()
    lg = _case(N, K, N + K)[0]
    seed, step = 4242 + K, 17
    d_lg = _dev(lg)
    act, pd = torch.zeros(N, K, device=DEV), torch.zeros(N, 2 * K, device=DEV)
    idx = torch.full((N,), -1, dtype=torch.int64, device=DEV)
    ctr = torch.tensor([step], dtype=torch.int64, device=DEV)
    assert L.sb200_ppo_cat_sample_f32(_p(d_lg), K, N, K, 0, seed, _p(ctr), _p(act), _p(pd), _p(idx), None, 0, None) == 0
    torch.cuda.synchronize()
    prob = PD.cat_prob(torch.tensor(lg, dtype=torch.float64)).numpy()
    u = agent_uniform(seed, step, np.arange(N))
    exp = PD.cat_sample(prob, K, u)
    c = np.cumsum(prob[:, :K], axis=1)
    safe = (np.abs(c - u[:, None]) > 1e-6).all(axis=1)
    got = idx.cpu().numpy()
    boundary = int((~safe).sum())
    print('sampler N=%d K=%d: %d boundary cases of %d' % (N, K, boundary, N))
    # each of the K boundaries excludes a 2e-6 wide band of u: about 2e-6 * K * N rows are expected there
    assert boundary <= 3 + int(4 * 2e-6 * K * N)
    assert np.array_equal(got[safe], exp[safe])
    assert np.array_equal(act.cpu().numpy().argmax(1), got) and bool((act.sum(1) == 1).all())
    _close(pd.cpu().numpy()[:, :K], prob[:, :K], 'sampled pd')
    # deterministic: the argmax (lowest index among ties)
    assert L.sb200_ppo_cat_sample_f32(_p(d_lg), K, N, K, 1, seed, _p(ctr), _p(act), _p(pd), _p(idx), None, 0, None) == 0
    torch.cuda.synchronize()
    assert np.array_equal(idx.cpu().numpy(), np.asarray(lg).argmax(1))


def test_sampler_chi_square_over_a_million_draws():
    from scipy.stats import chisquare
    L = _lib()
    K, N = 18, 1 << 20
    rng = np.random.default_rng(3)
    row = (rng.standard_normal(K) * 1.5).astype(np.float32)
    d_lg = _dev(np.tile(row, (N, 1)))
    act, pd = torch.zeros(N, K, device=DEV), torch.zeros(N, 2 * K, device=DEV)
    idx = torch.zeros(N, dtype=torch.int64, device=DEV)
    ctr = torch.tensor([5], dtype=torch.int64, device=DEV)
    assert L.sb200_ppo_cat_sample_f32(_p(d_lg), K, N, K, 0, 99, _p(ctr), _p(act), _p(pd), _p(idx), None, 0, None) == 0
    counts = np.bincount(idx.cpu().numpy(), minlength=K)
    p = PD.cat_prob(torch.tensor(row[None], dtype=torch.float64)).numpy()[0, :K]
    stat, pval = chisquare(counts, p * N)
    print('chi-square over %d draws, K=%d: %.2f (p = %.3f)' % (N, K, stat, pval))
    assert pval > 1e-3


# -- helpers for the agent / learner tests -----------------------------------------------------------------------------
def _cat_cfg(D, K, n, B, mode, actor_h=(32, 24), critic_h=(28, 20), lr=3e-3, rnn_layers=0, H=16, horizon=None, N=None):
    lc, ec, sc = ppo_configs(D=D, A=K, actor_h=actor_h, critic_h=critic_h, n_step=n, stride=n, B=B, mode=mode, lr=lr,
                             exp_interval=B)
    ec.action_spec = {'dim': (K,), 'type': 'discrete'}
    if rnn_layers:
        lc.algo.rnn.if_rnn_policy = True
        lc.algo.rnn.rnn_layer = rnn_layers
        lc.algo.rnn.rnn_hidden = H
        lc.algo.rnn.horizon = horizon
    if N is not None:
        ec.num_envs = N
    return lc, ec, sc


def _learner(lc, ec, sc, graph):
    from surreal_b200.learner import PPOLearner
    L = PPOLearner(lc, ec, sc)
    L.use_cuda_graph = graph
    return L


def _heads(sd, n_act, n_crit):
    al = [(sd['actor.model.seq.%d.weight' % (2 * i)], sd['actor.model.seq.%d.bias' % (2 * i)]) for i in range(n_act)]
    cl = [(sd['critic.model.seq.%d.weight' % (2 * i)], sd['critic.model.seq.%d.bias' % (2 * i)]) for i in range(n_crit)]
    return al, cl


def _batch(O, B, n, D, K, rng, cells=None):
    """Windows whose behaviour policy is the oracle's current policy on perturbed observations: one-hot actions drawn
    from it, pd rows [p | log p]."""
    obs = (rng.standard_normal((B, n, D)) * 1.2).astype(np.float32)
    obs_next = (rng.standard_normal((B, 1, D)) * 1.2).astype(np.float32)
    with torch.no_grad():
        if cells is not None:
            O.cells = tuple(torch.tensor(c, dtype=torch.float64).transpose(0, 1).contiguous() for c in cells)
        x = torch.tensor(obs + rng.standard_normal(obs.shape).astype(np.float32) * 0.1, dtype=torch.float64)
        pd = O.forward_actor(x if cells is not None else x.view(B * n, D)).reshape(B, n, 2 * K).numpy().astype(np.float32)
    idx = PD.cat_sample(pd.reshape(-1, 2 * K), K, rng.random(B * n)).reshape(B, n)
    actions = np.eye(K, dtype=np.float32)[idx]
    rewards = (rng.standard_normal((B, n)) * 0.3).astype(np.float32)
    dones = np.zeros((B, n), dtype=np.float32)
    dones[rng.random(B) < 0.3, n - 1] = 1
    return dict(obs=obs, obs_next=obs_next, actions=actions, rewards=rewards, dones=dones, pd=pd)


def _device_batch(b, cells=None):
    d = {'obs': {'low_dim': {'flat_inputs': b['obs']}}, 'obs_next': {'low_dim': {'flat_inputs': b['obs_next']}},
         'actions': b['actions'], 'rewards': b['rewards'], 'dones': b['dones'], 'persistent_infos': [b['pd']],
         'onetime_infos': cells}
    return d


STAT_KEYS = ['_surr_loss', '_clip_surr_loss', '_kl_loss_adapt', '_entropy', '_pol_kl', '_val_loss', '_avg_return_targ',
             '_avg_behave_likelihood', '_avg_is_weight', '_ref_behave_diff']


def _compare_learn(L, O, batches, host_batches, params):
    for it, (b, hb) in enumerate(zip(batches, host_batches)):
        st = L.learn(b)
        L.publish_parameter(it)
        st_o = O.learn(hb)
        O.publish_parameter()
        torch.cuda.synchronize()
        assert '_avg_log_sig' not in st
        assert L.last_n_policy_epochs == O.n_policy_epochs[-1], ('epochs', it)
        for k in STAT_KEYS:
            if k in st_o:
                assert abs(st[k] - st_o[k]) <= 1e-5 * max(1.0, abs(st_o[k])), (it, k, st[k], st_o[k])
    got, exp = params()
    d = torch.cat([(g.cpu().double() - e.detach().double()).abs().view(-1) for g, e in zip(got, exp)])
    lr = L.lr_actor
    assert float(d.median()) <= 0.002 * lr and float(d.pow(2).mean().sqrt()) <= 0.1 * lr, float(d.max())


# -- 4. learn() against the float64 oracle -------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', ['clip', 'adapt'])
@pytest.mark.parametrize('K', [3, 18])
def test_learn_mlp_matches_float64_oracle(mode, K):
    from cat_ref import CatOraclePPOLearner
    from oracle.filters import ZFilter as OZ
    D, n, B = 11, 4, 64
    lc, ec, sc = _cat_cfg(D, K, n, B, mode)
    L = _learner(lc, ec, sc, graph=True)
    assert L.categorical and L.model.log_var is None and L._epoch_kernels() is None
    rng = np.random.default_rng(K)
    zf = OZ(D)
    zf.update(torch.randn(300, D, generator=torch.Generator().manual_seed(1)) * 1.3)
    L.model.z_stats.copy_(torch.cat([zf.running_sum, zf.running_sumsq, zf.count]).to(DEV))
    L.ref_target_model.update_target_params(L.model)
    sd = {k: v.cpu() for k, v in L.model.state_dict().items()}
    al, cl = _heads(sd, 3, 3)
    O = CatOraclePPOLearner(al, cl, zf, K, n, B, ppo_mode=mode, lr_actor=lc.algo.network.lr_actor,
                            lr_critic=lc.algo.network.lr_critic, exp_interval=B)
    hbs = [_batch(O, B, n, D, K, rng) for _ in range(3)]
    _compare_learn(L, O, [_device_batch(b) for b in hbs], hbs,
                   lambda: ([t for l in range(3) for t in L.model.actor.get_layer(l)],
                            [t for wb in O.actor for t in wb]))


@pytest.mark.parametrize('mode', ['clip', 'adapt'])
@pytest.mark.parametrize('layers', [1, 2])
def test_learn_lstm_matches_float64_oracle(mode, layers):
    from cat_ref import CatOraclePPOLearnerRNN
    from oracle.filters import ZFilter as OZ
    D, K, n, B, H, hz = 9, 6, 6, 16, 16, 3
    lc, ec, sc = _cat_cfg(D, K, n, B, mode, rnn_layers=layers, H=H, horizon=hz)
    L = _learner(lc, ec, sc, graph=True)
    rng = np.random.default_rng(layers)
    sd = {k: v.cpu() for k, v in L.model.state_dict().items()}
    al, cl = _heads(sd, 3, 3)
    lstm = {k.split('.', 1)[1]: sd[k] for k in sd if k.startswith('rnn_stem.')}
    zf = OZ(D).load(sd['z_filter.running_sum'], sd['z_filter.running_sumsq'], sd['z_filter.count'])
    O = CatOraclePPOLearnerRNN(al, cl, zf, lstm, K, n, B, hz, H, layers, ppo_mode=mode,
                               lr_actor=lc.algo.network.lr_actor, lr_critic=lc.algo.network.lr_critic, exp_interval=B)
    hbs, dbs = [], []
    for _ in range(3):
        cells = [(rng.standard_normal((B, layers, H)) * 0.3).astype(np.float32) for _ in range(2)]
        b = _batch(O, B, n, D, K, rng, cells=cells)
        b['h0'], b['c0'] = cells
        hbs.append(b)
        dbs.append(_device_batch(b, cells=cells))
    _compare_learn(L, O, dbs, hbs, lambda: ([t for l in range(3) for t in L.model.actor.get_layer(l)],
                                           [t for wb in O.actor for t in wb]))


@pytest.mark.parametrize('mode', ['clip', 'adapt'])
def test_learn_cnn_matches_float64_oracle(mode):
    from cat_ref import CatOraclePPOLearnerPixel
    C, HW, Fd, K, n, B = 4, 28, 24, 5, 3, 16
    # lr of the existing pixel learner tests: Adam turns fp32-vs-fp64 noise on the CNN's near-zero gradients into whole
    # steps, which at larger rates moves the value loss of later epochs beyond the learner tolerance
    lc, ec, sc = _cat_cfg(1, K, n, B, mode, lr=1e-4)
    lc.algo.use_z_filter = False
    ec.obs_spec = {'pixel': {'camera0': (C, HW, HW)}}
    ec.pixel_input = True
    lc.model.cnn_feature_dim = Fd
    L = _learner(lc, ec, sc, graph=True)
    sd = {k: v.cpu() for k, v in L.model.state_dict().items()}
    conv = [(sd['cnn_stem.model.seq.0.weight'], sd['cnn_stem.model.seq.0.bias']),
            (sd['cnn_stem.model.seq.2.weight'], sd['cnn_stem.model.seq.2.bias'])]
    fc = (sd['cnn_stem.model.seq.5.weight'], sd['cnn_stem.model.seq.5.bias'])
    al, cl = _heads(sd, 3, 3)
    O = CatOraclePPOLearnerPixel(al, cl, conv, [4, 2], fc, K, n, B, ppo_mode=mode, lr_actor=lc.algo.network.lr_actor,
                                 lr_critic=lc.algo.network.lr_critic, exp_interval=B)
    rng = np.random.default_rng(5)
    hbs, dbs = [], []
    for _ in range(2):
        fr = rng.integers(0, 256, (B, n + 1, C, HW, HW)).astype(np.uint8)
        with torch.no_grad():
            pd = O.forward_actor(torch.tensor(fr[:, :n].reshape(-1, C, HW, HW), dtype=torch.float64)).numpy()
        pd = pd.reshape(B, n, 2 * K).astype(np.float32)
        idx = PD.cat_sample(pd.reshape(-1, 2 * K), K, rng.random(B * n)).reshape(B, n)
        b = dict(obs=fr[:, :n], obs_next=fr[:, n:], actions=np.eye(K, dtype=np.float32)[idx],
                 rewards=(rng.standard_normal((B, n)) * 0.3).astype(np.float32), dones=np.zeros((B, n), np.float32), pd=pd)
        hbs.append(dict(b, obs=b['obs'].astype(np.float32), obs_next=b['obs_next'].astype(np.float32)))
        dbs.append({'obs': {'pixel': {'camera0': b['obs']}}, 'obs_next': {'pixel': {'camera0': b['obs_next']}},
                    'actions': b['actions'], 'rewards': b['rewards'], 'dones': b['dones'], 'persistent_infos': [pd],
                    'onetime_infos': None})
    _compare_learn(L, O, dbs, hbs, lambda: ([t for l in range(3) for t in L.model.actor.get_layer(l)],
                                           [t for wb in O.actor for t in wb]))


@pytest.mark.parametrize('rnn', [0, 1])
def test_graph_replay_is_bitwise_equal_to_eager(rnn):
    D, K, n, B = 11, 18, 6, 64
    kw = dict(rnn_layers=1, H=16, horizon=3) if rnn else {}
    out = []
    for graph in (True, False):
        lc, ec, sc = _cat_cfg(D, K, n, B, 'adapt', **kw)
        torch.manual_seed(0)
        L = _learner(lc, ec, sc, graph=graph)
        if out:
            L.model.load_state_dict(out[0][0])
            L.ref_target_model.update_target_params(L.model)
        sd0 = {k: v.clone() for k, v in L.model.state_dict().items()}
        rng = np.random.default_rng(9)
        for it in range(3):
            pd = PD.cat_prob(torch.tensor(rng.standard_normal((B * n, K)))).numpy().astype(np.float32).reshape(B, n, 2 * K)
            b = dict(obs=rng.standard_normal((B, n, D)).astype(np.float32), obs_next=rng.standard_normal((B, 1, D)).astype(np.float32),
                     actions=np.eye(K, dtype=np.float32)[rng.integers(0, K, (B, n))], rewards=rng.standard_normal((B, n)).astype(np.float32),
                     dones=np.zeros((B, n), np.float32), pd=pd)
            cells = [np.zeros((B, 1, 16), np.float32)] * 2 if rnn else None
            L.learn(_device_batch(b, cells))
            L.publish_parameter(it)
        torch.cuda.synchronize()
        out.append((sd0, L.model.actor.params.clone(), L.model.critic.params.clone(), L._stats.clone()))
    assert torch.equal(out[0][1], out[1][1]) and torch.equal(out[0][2], out[1][2]) and torch.equal(out[0][3], out[1][3])


# -- 3. staging: act() + DiscreteSyntheticEnv through ppo_window_step ---------------------------------------------------
def test_act_and_discrete_env_stage_the_oracle_windows():
    from oracle.windowing import multistep_windows
    from surreal_b200.agent import PPOAgent
    from surreal_b200.replay import FIFOReplay
    from surreal_b200.env import DiscreteSyntheticEnv
    N, D, K, n, stride, cap = 24, 8, 5, 4, 2, 7
    lc, ec, sc = _cat_cfg(D, K, n, 64, 'clip', N=N)
    lc.algo.stride = stride
    lc.replay.memory_size = 4096
    R = FIFOReplay(lc, ec, sc)
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    assert ag.categorical and not ag.rollout_chunk_supported()
    env = DiscreteSyntheticEnv(N, D, K, limit_episode_length=cap, seed=2)
    ag.env = w = ag.prepare_env_agent(env)
    obs, _ = w.reset()
    ep0 = np.arange(N) % cap                                        # staggered episodes
    env.ep_step.copy_(torch.tensor(ep0, dtype=torch.int32))
    T = 20
    rec = {k: [] for k in ('obs', 'act', 'pd', 'rew', 'done', 'next')}
    for t in range(T):
        rec['obs'].append(obs['low_dim']['flat_inputs'].clone())
        a = ag.act(obs)
        assert a[0].shape == (N, K) and bool((a[0].sum(1) == 1).all())
        rec['act'].append(a[0].clone())
        rec['pd'].append(a[1][1][0].clone())
        obs, rew, done, info = w.step(a)
        rec['rew'].append(rew.clone())
        rec['done'].append(done.clone())
        rec['next'].append(info['obs_next'].clone())
    torch.cuda.synchronize()
    S = {k: torch.stack(v, 1).cpu().numpy() for k, v in rec.items()}        # [N, T, ...]
    # the oracle's windows per actor, in (completion step, actor) arrival order
    expect = []
    for i in range(N):
        first = cap - ep0[i]
        lens = [first] + [cap] * ((T - first) // cap + 1)
        for ids, nxt, dn in multistep_windows(lens, n, stride):
            if ids[-1] < T:
                expect.append((ids[-1], i, ids, dn))
    expect.sort(key=lambda e: (e[0], e[1]))
    assert len(R) == len(expect) > 0
    b = R.sample(len(expect))
    got = {k: v.cpu().numpy() for k, v in (('obs', b['obs']['low_dim']['flat_inputs']), ('next', b['obs_next']['low_dim']['flat_inputs']),
                                           ('act', b['actions']), ('pd', b['persistent_infos'][0]), ('rew', b['rewards']),
                                           ('done', b['dones']))}
    for r, (_, i, ids, dn) in enumerate(expect):
        assert np.array_equal(got['obs'][r], S['obs'][i, ids]), r
        assert np.array_equal(got['next'][r, 0], S['next'][i, ids[-1]]), r
        assert np.array_equal(got['act'][r], S['act'][i, ids]) and np.array_equal(got['pd'][r], S['pd'][i, ids]), r
        assert np.array_equal(got['rew'][r], S['rew'][i, ids]) and np.array_equal(got['done'][r], np.asarray(dn, np.float32)), r
    # the behaviour pd rows are the oracle's softmax of the actor head, and the actions its Philox inverse-CDF draws
    sd = {k: v.cpu() for k, v in ag.model.state_dict().items()}
    al, _ = _heads(sd, 3, 3)
    from oracle.nets import mlp_trunk
    from oracle.filters import ZFilter as OZ
    zf = OZ(D).load(sd['z_filter.running_sum'], sd['z_filter.running_sumsq'], sd['z_filter.count'])
    x = zf.forward(torch.tensor(S['obs'][:, 0], dtype=torch.float64))
    prob = PD.cat_prob(mlp_trunk(x, [(w_.double(), b_.double()) for w_, b_ in al])).detach().numpy()
    _close(S['pd'][:, 0], prob, 'behaviour pd')
    u = agent_uniform(ag.seed, 0, np.arange(N))
    c = np.cumsum(prob[:, :K], axis=1)
    safe = (np.abs(c - u[:, None]) > 1e-6).all(axis=1)
    assert np.array_equal(S['act'][:, 0].argmax(1)[safe], PD.cat_sample(prob, K, u)[safe])


def test_act_host_observations_give_indices_and_eval_is_argmax():
    from surreal_b200.agent import PPOAgent
    N, D, K = 8, 6, 7
    lc, ec, sc = _cat_cfg(D, K, 4, 16, 'clip', N=N)
    ag = PPOAgent(lc, ec, sc, 0, 'eval_deterministic_local')
    x = np.random.default_rng(0).standard_normal((N, D)).astype(np.float32)
    a = ag.act(x)
    assert a.dtype == np.int64 and a.shape == (N,)
    with torch.no_grad():
        pd = ag.model.forward_actor(torch.tensor(x, device=DEV)).cpu().numpy()
    assert np.array_equal(a, pd[:, :K].argmax(1))
    dev = ag.act(torch.tensor(x, device=DEV))
    assert torch.equal(dev.argmax(1).cpu(), torch.tensor(a))


# -- 5. checkpoints ---------------------------------------------------------------------------------------------------
def test_checkpoint_round_trip_and_cross_type_load_error():
    from surreal_b200.model.ppo_net import PPOModel
    lc, ec, sc = _cat_cfg(11, 18, 4, 16, 'clip')
    mk = dict(obs_spec=ec.obs_spec, action_dim=18, model_config=lc.model, use_z_filter=True, rnn_config=lc.algo.rnn)
    a = PPOModel(categorical=True, **mk)
    for l in range(a.actor.n_layers):
        w, bias = a.actor.get_layer(l)
        a.actor.set_layer(l, torch.rand_like(w) * 2 - 1, torch.rand_like(bias) * 2 - 1)
    sd = a.state_dict()
    assert 'actor.log_var' not in sd
    b = PPOModel(categorical=True, **mk)
    b.load_state_dict(copy.deepcopy({k: v.cpu() for k, v in sd.items()}))
    assert torch.equal(a.actor.params, b.actor.params) and torch.equal(a.critic.params, b.critic.params)
    assert all(torch.equal(v, b.state_dict()[k]) for k, v in sd.items())
    g = PPOModel(categorical=False, **mk)
    with pytest.raises(ValueError, match='categorical'):
        g.load_state_dict(sd)
    with pytest.raises(ValueError, match='Gaussian'):
        b.load_state_dict(g.state_dict())

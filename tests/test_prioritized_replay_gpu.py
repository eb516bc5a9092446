"""PrioritizedReplay on the GPU against its float64 restatement (per_ref.py): the trees after host inserts, wrapping
device chunks and priority updates; the proportional sampler against the descent over the device's own leaves; the
distribution of a million draws; weights and the beta schedule inside one graph; the last-wins and stop-flag rules of
the write-back; the weighted learner against hand-driven updates and float64 autograd; the engine and the launcher."""
import numpy as np
import pytest
import torch

from helpers import ddpg_configs
from per_ref import PerRef, TreeRef, beta_schedule, leaf_value, philox_u
from test_ddpg_device_engine_gpu import STAT_KEYS, _SequenceEnv, _learner_state, _nan_out

pytestmark = pytest.mark.gpu

FIELDS = ('obs', 'obs_next', 'actions', 'rewards', 'dones')


def _per(capacity, D=12, A=4, B=64, sampler_seed=7, fill=True, n_step=3, **rc):
    from surreal_b200.replay import PrioritizedReplay
    lc, ec, sc = ddpg_configs(D=D, A=A, B=B, memory_size=capacity, start=0, n_step=n_step)
    lc.replay.sampler_seed = sampler_seed
    for k, v in rc.items():
        lc.replay[k] = v
    r = PrioritizedReplay(lc, ec, sc)
    if fill:
        g = torch.Generator(device='cuda').manual_seed(capacity)
        for t in (r.r_obs, r.r_obs_next, r.r_rew):
            t.normal_(generator=g)
        r.r_act.uniform_(-1, 1, generator=g)
    return r, (lc, ec, sc)


def _fill_ring(r, seed, decades=4):
    """Every slot admitted, then random priorities 10^U(-decades/2, decades/2) set through the host path."""
    C_ = r.memory_size
    r.state.copy_(torch.tensor([0, C_, C_, C_]))
    r._dirty = True
    r.admit()
    rng = np.random.RandomState(seed)
    p = (10.0 ** rng.uniform(-decades / 2, decades / 2, size=C_)).astype(np.float32)
    r.update_priorities(np.arange(C_), p)
    return p


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _check_trees(r, ref):
    leaf = r.t_leaf.cpu().numpy()
    assert _ulps(leaf[:r.memory_size], ref.tree.leaf[:r.memory_size]).max() <= 2
    assert (leaf[r.memory_size:] == 0).all()
    dev = TreeRef(r.memory_size, leaf)                         # internal nodes against float64 over the device's leaves
    s = r.t_sum.cpu().numpy()
    assert np.allclose(s[1:], dev.sum[1:], rtol=1e-12, atol=0)
    assert np.array_equal(r.t_min.cpu().numpy()[1:], dev.mn[1:])
    assert r.max_priority == float(ref.max_priority)
    assert (r.t_owner == -1).all() and (r.t_dirty == 0).all()


# ---- trees ----------------------------------------------------------------------------------------------------------
def test_trees_after_inserts_wrapping_chunks_and_updates():
    from surreal_b200.env import ExpSenderWrapperSSARNStepBootstrap
    N, D, A, C_ = 64, 12, 4, 1000
    r, (lc, ec, sc) = _per(C_, D=D, A=A, n_step=1, fill=False, alpha=0.7)
    ref = PerRef(C_, 0.7)
    rng = np.random.RandomState(0)
    for _ in range(5):                                         # host inserts
        o = {'low_dim': {'flat_inputs': rng.randn(D).astype(np.float32)}}
        r.insert({'obs': [o, o], 'action': rng.randn(A).astype(np.float32), 'reward': 1.0, 'done': 0.0})
    r.snapshot_view()
    ref.admit(5)
    _check_trees(r, ref)
    idx, p = np.array([0, 3, 0, 4, 3]), np.array([2.5, 0.1, 0.7, 3.0, 9.0], np.float32)
    r.update_priorities(idx, p)
    ref.update(idx, p)
    _check_trees(r, ref)
    env = ExpSenderWrapperSSARNStepBootstrap(_SequenceEnv(N, D, A), lc, sc, replay=r)
    env.reset()
    act = torch.zeros(N, A, device='cuda')
    total = 5
    for chunk in range(4):                                     # 640 records a chunk: the ring wraps from the second on
        for _ in range(10):
            env.step(act)
        total += 10 * N
        r.snapshot_view(reserve=N * 10)
        ref.admit(total)
        _check_trees(r, ref)
        k = 300
        idx = rng.randint(0, C_, size=k)
        idx[-20:] = idx[:20]                                   # duplicates: the later value stays
        p = (10.0 ** rng.uniform(-3, 1, size=k)).astype(np.float32)
        p[chunk] = 11.0 + chunk                                # max_priority goes up
        r.update_priorities_device(torch.from_numpy(idx).cuda(), torch.from_numpy(p).cuda())
        ref.update(idx, p)
        _check_trees(r, ref)
    assert int(r.state[3]) == total and int(r.ctrl[0]) == total


# ---- sampler --------------------------------------------------------------------------------------------------------
def _compare_draws(r, start, count, seed, ctr, B, beta):
    full, out = _nan_out(r, B)
    batch = r.sample_device(B, out=out)
    torch.cuda.synchronize()
    t = TreeRef(r.memory_size, r.t_leaf.cpu().numpy())
    want, masses, S = t.sample(start, count, philox_u(seed, ctr, B))
    got = batch['indices'].cpu().numpy()
    bad = np.nonzero(got != want)[0]
    if len(bad):
        bounds = t.prefix_boundaries(start, count)
        for b in bad:                                          # only draws at a prefix boundary may round the other way
            assert np.abs(bounds - masses[b]).min() <= 1e-9 * S, (b, got[b], want[b])
        assert len(bad) <= B * 1e-5
    assert ((got - start) % r.memory_size < count).all() and (t.leaf[got] > 0).all()
    w = batch['weights'].cpu().numpy()[:, 0]
    assert batch['weights'].shape == (B, 1)
    assert np.allclose(w, t.weights(got, start, count, beta), rtol=1e-6, atol=0)
    assert torch.equal(batch['actions'], r.r_act[batch['indices']])
    assert torch.equal(batch['obs']['low_dim']['flat_inputs'], r.r_obs[batch['indices']])
    for k in FIELDS:
        assert torch.isnan(full[k][B:]).all()
    return got


@pytest.mark.parametrize('cap', [1000, 2 ** 20 + 8])
def test_sampler_matches_the_descent_over_the_device_leaves(cap):
    seed, ctr, B = 99, 12, 4097
    r, _ = _per(cap, sampler_seed=seed, beta0=0.5, beta_anneal_iters=10)
    _fill_ring(r, cap)
    r.ctrl[1] = 3
    for start, count in ((0, cap), (0, cap // 3), (cap - 3, cap - 10), (cap // 2, cap // 2 + 7)):
        r.view.copy_(torch.tensor([start, count, cap]))
        r.sampler[0] = ctr
        t0 = r.update_counter
        _compare_draws(r, start, count, seed, ctr, B, beta_schedule(t0, 0.5, 10))
        assert r.draw_counter == ctr + 1 and r.update_counter == t0 + 1 and r.sampler_status == 0
        ctr += 1


def test_sampler_on_an_empty_view_touches_nothing():
    r, _ = _per(256)
    _fill_ring(r, 1)
    r.view.copy_(torch.tensor([0, 0, 256]))
    r.sampler[0] = 9
    full, out = _nan_out(r, 64)
    idx0, w0 = r._dev_indices.clone(), r._dev_weights.clone()
    r.sample_device(64, out=out)
    torch.cuda.synchronize()
    assert r.sampler_status == 1 and r.draw_counter == 9 and r.update_counter == 0
    assert all(torch.isnan(v).all() for v in full.values())
    assert torch.equal(r._dev_indices, idx0) and torch.equal(r._dev_weights, w0)


def test_a_million_draws_follow_the_priorities():
    from scipy.stats import chi2
    r, _ = _per(1000, B=2 ** 16, sampler_seed=2024)
    _fill_ring(r, 5, decades=4)
    r.view.copy_(torch.tensor([0, 1000, 1000]))
    hist = torch.zeros(1000, dtype=torch.int64, device='cuda')
    for _ in range(16):                                        # 16 x 65536 draws
        b = r.sample_device(2 ** 16)
        hist += torch.bincount(b['indices'], minlength=1000)
    leaf = r.t_leaf[:1000].double().cpu().numpy()
    n = float(hist.sum())
    expect = n * leaf / leaf.sum()
    stat = float(((hist.cpu().numpy() - expect) ** 2 / expect).sum())
    assert stat < chi2.ppf(1 - 1e-3, 999), stat


def test_weights_and_beta_step_inside_one_graph():
    from surreal_b200 import _lib
    seed, B, K = 5, 256, 8
    r, _ = _per(3000, B=B, sampler_seed=seed, beta0=0.4, beta_anneal_iters=5)
    _fill_ring(r, 3)
    r.view.copy_(torch.tensor([2500, 2000, 3000]))
    r.sampler[0], r.ctrl[1] = 40, 1
    keep_w = torch.zeros(K, B, device='cuda')
    keep_i = torch.zeros(K, B, dtype=torch.int64, device='cuda')
    _lib.ensure_device()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for k in range(K):
            b = r.sample_device(B)
            keep_w[k].copy_(b['weights'][:, 0])
            keep_i[k].copy_(b['indices'])
    for rep in range(2):
        g.replay()
        torch.cuda.synchronize()
        t = TreeRef(3000, r.t_leaf.cpu().numpy())
        for k in range(K):
            step = 1 + rep * K + k
            want, _, _ = t.sample(2500, 2000, philox_u(seed, 40 + rep * K + k, B))
            got = keep_i[k].cpu().numpy()
            assert (got == want).mean() > 0.999
            beta = beta_schedule(step, 0.4, 5)
            assert np.allclose(keep_w[k].cpu().numpy(), t.weights(got, 2500, 2000, beta), rtol=1e-6, atol=0)
    assert r.update_counter == 1 + 2 * K


# ---- write-back -----------------------------------------------------------------------------------------------------
def test_duplicates_take_the_last_value_and_a_stop_flag_changes_nothing():
    r, _ = _per(500, alpha=0.6)
    _fill_ring(r, 4)
    ref = PerRef(500, 0.6)
    ref.tree.leaf[:500] = r.t_leaf[:500].cpu().numpy()
    ref.max_priority = np.float32(r.max_priority)
    idx = torch.tensor([7, 9, 7, 7, 300, 9, 499], device='cuda')
    p = torch.tensor([1.0, 2.0, 3.0, 0.25, 5.0, 0.5, 1000.0], device='cuda')
    stop = torch.ones(1, dtype=torch.int32, device='cuda')
    before = [t.clone() for t in (r.t_leaf, r.t_sum, r.t_min, r.ctrl)]
    r.update_priorities_device(idx, p, stop_flag=stop)
    torch.cuda.synchronize()
    for a, b in zip(before, (r.t_leaf, r.t_sum, r.t_min, r.ctrl)):
        assert torch.equal(a, b)
    stop.zero_()
    r.update_priorities_device(idx, p, stop_flag=stop)
    ref.update(idx.cpu().numpy(), p.cpu().numpy())
    assert r.t_leaf[7] == float(leaf_value(0.25, 0.6)) and r.t_leaf[9] == float(leaf_value(0.5, 0.6))
    _check_trees(r, ref)
    with pytest.raises(AssertionError):
        r.update_priorities([3], [0.0])
    with pytest.raises(AssertionError):
        r.update_priorities([500], [1.0])


# ---- learner --------------------------------------------------------------------------------------------------------
def _tree_state(r):
    return [t.clone() for t in (r.t_leaf, r.t_sum, r.t_min, r.ctrl, r.sampler)]


def _restore(r, snap):
    for t, s in zip((r.t_leaf, r.t_sum, r.t_min, r.ctrl, r.sampler), snap):
        t.copy_(s)


def _twin(target, graphs=True, layernorm=False, td3=False, alpha=0.6):
    from surreal_b200.learner import DDPGLearner
    r, _ = _per(600, D=9, A=3, B=16, sampler_seed=3, alpha=alpha, beta_anneal_iters=7)
    _fill_ring(r, 6)
    r.view.copy_(torch.tensor([590, 500, 600]))
    out = []
    for _ in range(2):
        lc, ec, sc = ddpg_configs(D=9, A=3, B=16, target=dict(target))
        lc.model.use_layernorm = layernorm
        lc.algo.network.use_double_critic = lc.algo.network.use_action_regularization = td3
        lc.algo.network.critic_regularization = 1e-3
        torch.manual_seed(11)
        out.append(DDPGLearner(lc, ec, sc))
    out[0].use_cuda_graph = graphs
    return r, out[0], out[1]


@pytest.mark.parametrize('case', ['hard', 'soft', 'td3', 'layernorm', 'graphs_off'])
def test_learn_from_replay_equals_k_hand_driven_updates(case):
    target = {'type': 'soft', 'tau': 0.05, 'interval': 1} if case == 'soft' else {'type': 'hard', 'interval': 3}
    r, LA, LB = _twin(target, graphs=case != 'graphs_off', layernorm=case == 'layernorm', td3=case == 'td3')
    K = 5
    for call in range(2):
        snap = _tree_state(r)
        sa = LA.learn_from_replay(r, updates=K)
        after = _tree_state(r)
        _restore(r, snap)
        for _ in range(K):
            b = r.sample_device(16, out=LB.replay_out_buffers())
            sb = LB.learn(b)
            r.update_priorities(b['indices'], LB.td_priorities)
        torch.cuda.synchronize()
        for a, b_ in zip(after, _tree_state(r)):
            assert torch.equal(a, b_)
        for a, b_ in zip(_learner_state(LA), _learner_state(LB)):
            assert torch.equal(a, b_)
        for k in STAT_KEYS + ('td_error', 'avg_is_weight') + (('Q_policy2',) if case == 'td3' else ()):
            assert sa[k] == sb[k], k
        assert 0 < sa['avg_is_weight'] <= 1 and sa['td_error'] > 0
    assert not np.all(r.priorities()[:600] == r.priorities()[0])


def test_learn_writes_priorities_to_the_attached_replay():
    r, LA, _ = _twin({'type': 'hard', 'interval': 3})
    LA.attach_replay(r)
    r.ctrl[1] = 0
    b = r.sample(16)
    before = r.priorities().copy()
    LA.learn(b)
    torch.cuda.synchronize()
    ref = PerRef(600, r.alpha)
    ref.tree.leaf[:600] = before
    ref.update(b['indices'].cpu().numpy(), LA.td_priorities.cpu().numpy())
    assert _ulps(r.priorities(), ref.tree.leaf[:600]).max() <= 2


def test_weighted_critic_gradient_matches_float64_autograd():
    from surreal_b200 import _lib
    L = _lib.lib()
    B, eps = 777, 1e-6
    g = torch.Generator(device='cuda').manual_seed(1)
    q = torch.randn(B, 1, device='cuda', generator=g)
    y = torch.randn(B, device='cuda', generator=g)
    w = torch.rand(B, device='cuda', generator=g) + 0.05
    dq = torch.full((B, 4), float('nan'), device='cuda')
    prio = torch.zeros(B, device='cuda')
    stats = torch.zeros(16, device='cuda')
    ws = torch.zeros(L.sb200_ddpg_workspace_bytes(B), dtype=torch.uint8, device='cuda')
    p = lambda t: t.data_ptr()  # noqa: E731
    from surreal_b200.ops import _stream
    assert L.sb200_ddpg_critic_loss_weighted_f32(p(q), 1, p(y), B, p(w), p(dq), 4, p(prio), eps, p(stats), p(ws),
                                                 _stream()) == 0
    torch.cuda.synchronize()
    q64 = q.double().clone().requires_grad_(True)
    d = q64[:, 0] - y.double()
    loss = (w.double() * d ** 2).mean()
    loss.backward()
    assert torch.allclose(dq[:, 0].double(), q64.grad[:, 0], rtol=1e-6, atol=1e-12)
    assert (dq[:, 1:] == 0).all()
    assert abs(float(stats[1]) - loss.item()) <= 1e-6 * loss.item()
    assert abs(float(stats[7]) - float(d.abs().mean())) <= 1e-6 * float(d.abs().mean())
    assert abs(float(stats[8]) - float(w.double().mean())) <= 1e-6
    assert torch.allclose(prio.double(), (q[:, 0] - y).abs().double() + eps, rtol=1e-7, atol=0)


def test_alpha_zero_weights_are_one_and_the_update_is_the_uniform_one():
    r, LA, LB = _twin({'type': 'hard', 'interval': 3}, alpha=0.0)
    b = r.sample_device(16, out=LA.replay_out_buffers())
    torch.cuda.synchronize()
    assert (b['weights'] == 1).all()
    batch = {k: (v.clone() if isinstance(v, torch.Tensor) else
                 {'low_dim': {'flat_inputs': v['low_dim']['flat_inputs'].clone()}}) for k, v in b.items()}
    plain = {k: v for k, v in batch.items() if k not in ('weights', 'indices')}
    sa, sb = LA.learn(batch), LB.learn(plain)
    for a, b_ in zip(_learner_state(LA), _learner_state(LB)):
        assert torch.equal(a, b_)
    for k in STAT_KEYS:
        assert sa[k] == sb[k], k
    assert sa['avg_is_weight'] == 1.0 and 'td_error' not in sb


def test_bad_action_leaves_learner_and_priorities_untouched():
    r, LA, _ = _twin({'type': 'soft', 'tau': 0.01, 'interval': 1})
    LA.learn_from_replay(r, updates=3)
    snap, tree = _learner_state(LA), [t.clone() for t in (r.t_leaf, r.t_sum, r.t_min)]
    maxp = r.max_priority
    r.r_act[7, 1] = 1.5
    r.view.copy_(torch.tensor([7, 1, 600]))
    with pytest.raises(AssertionError):
        LA.learn_from_replay(r, updates=3)
    torch.cuda.synchronize()
    for a, b in zip(snap, _learner_state(LA)):
        assert torch.equal(a, b)
    for a, b in zip(tree, (r.t_leaf, r.t_sum, r.t_min)):
        assert torch.equal(a, b)
    assert r.max_priority == maxp


# ---- engine and launcher --------------------------------------------------------------------------------------------
def _run_engine(overlap, steps=14):
    from surreal_b200.launch import SurrealDefaultLauncher, ReplayEngine
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.learner import DDPGLearner
    from surreal_b200.replay import PrioritizedReplay
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    N, T, K = 32, 8, 4
    lc, ec, sc = ddpg_configs(D=12, A=4, actor_h=(48, 32), critic_h=(64, 48), B=64, n_step=3, memory_size=2000,
                              start=1000, target={'type': 'hard', 'interval': 7})
    lc.replay.beta_anneal_iters = 20
    make_synthetic_env_config(ec, N, 12, 4, seed=1)
    ec.num_agents = N
    ec.limit_episode_length = 20
    sc.agent.fetch_parameter_interval = 16
    lc.parameter_publish.min_publish_interval = 0
    torch.manual_seed(3)
    la = SurrealDefaultLauncher(DDPGAgent, DDPGLearner, PrioritizedReplay, sc, ec, lc)
    agent, replay, learner = la.setup_engine()
    eng = ReplayEngine(agent, replay, learner, T, K, overlap=overlap)
    eng.prime()
    stats = []
    for _ in range(steps):
        st = eng.step()
        if st is not None:
            stats.append([st[k] for k in STAT_KEYS + ('td_error', 'avg_is_weight')])
    eng.drain()
    assert len(stats) >= 3 and np.isfinite(np.array(stats)).all()
    state = [t.clone() for t in (replay.r_obs, replay.r_act, replay.state, replay.t_leaf, replay.t_sum, replay.t_min,
                                 replay.ctrl)]
    return state + _learner_state(learner), stats


def test_engine_two_streams_equal_the_one_stream_schedule():
    s2, stats2 = _run_engine(overlap=True)
    s1, stats1 = _run_engine(overlap=False)
    assert stats1 == stats2
    for a, b in zip(s1, s2):
        assert torch.equal(a, b)


def test_ddpg_launcher_trains_with_prioritized_replay(tmp_path):
    from surreal_b200.main.ddpg_configs import DDPGLauncher
    from surreal_b200.replay import PrioritizedReplay
    la = DDPGLauncher()
    learner = la.main(['learner', '--', '--env', 'synthetic:12:4', '--num-agents', '32', '--experiment-folder',
                       str(tmp_path), '--unit-test', '--prioritized-replay', '--rollout-steps', '8',
                       '--updates-per-chunk', '2', '--iterations', '4'])
    assert learner.current_iteration == 2 * 4
    assert isinstance(la.replay, PrioritizedReplay)
    n = len(la.replay)
    pr = la.replay.priorities()[:n]
    assert (pr > 0).all() and (pr != 1.0).any()

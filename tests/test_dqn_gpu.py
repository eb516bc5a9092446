"""DQN on the GPU: the act kernel (argmax, ties, epsilon, Philox replay, eval modes), the TD kernel against float64
autograd for every head form, DQNLearner against the float64 oracle across target copies, K graph updates against eager
ones, prioritized replay write-back, ReplayEngine on two streams against one, the host-env loop and checkpoints."""
import copy
import ctypes as C
import tempfile

import numpy as np
import pytest
import torch

from oracle import dqn as odqn

pytestmark = pytest.mark.gpu


def dqn_configs(D=10, n=5, hidden=(32, 24), B=64, dueling=True, double_q=True, period=100, lr=1e-3, memory_size=4096,
                start=200, steps=1000, clip=10.0, prioritized=False):
    from surreal_b200.session import Config
    from surreal_b200.main.dqn_configs import (DQN_DEFAULT_LEARNER_CONFIG, DQN_DEFAULT_ENV_CONFIG,
                                               DQN_DEFAULT_SESSION_CONFIG, make_discrete_synthetic_env_config)
    lc = Config(copy.deepcopy(DQN_DEFAULT_LEARNER_CONFIG.to_dict()))
    ec = Config(copy.deepcopy(DQN_DEFAULT_ENV_CONFIG.to_dict()))
    sc = Config(copy.deepcopy(DQN_DEFAULT_SESSION_CONFIG.to_dict()))
    sc.folder = tempfile.mkdtemp()
    make_discrete_synthetic_env_config(ec, 4, D, n, seed=1)
    ec.num_agents = 4
    lc.model.convs, lc.model.fc_hidden_sizes, lc.model.dueling = [], list(hidden), dueling
    lc.algo.double_q, lc.algo.target_network_update_freq, lc.algo.lr = double_q, period, lr
    lc.algo.grad_norm_clipping = clip
    lc.algo.exploration.steps = steps
    lc.algo.prioritized.enabled = prioritized
    lc.eval.eps = 0.05
    lc.replay.batch_size, lc.replay.memory_size, lc.replay.sampling_start_size = B, memory_size, start
    return lc, ec, sc


def _act(adv, val, eps=None, sched=None, seed=3, counter=0, one_hot=True):
    from surreal_b200 import _lib, ops
    N, n = adv.shape
    dev = adv.device
    action = torch.zeros(N, 1, device=dev)
    oh = torch.full((N, n + 3), 7.0, device=dev) if one_hot else None
    i64 = torch.zeros(N, dtype=torch.int64, device=dev)
    ctr = torch.tensor([counter], dtype=torch.int64, device=dev)
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    P = (sched.numel() - 1) // 2 if sched is not None else 0
    _lib.check(_lib.lib().sb200_dqn_act_f32(p(adv), adv.stride(0), p(val), 1, N, n, p(sched), P,
                                            0.0 if eps is None else eps, seed, p(ctr), p(action), p(oh),
                                            oh.stride(0) if oh is not None else 0, p(i64), ops._stream()), 'act')
    torch.cuda.synchronize()
    return action.view(-1).cpu().numpy(), (oh.cpu().numpy() if oh is not None else None), i64.cpu().numpy()


def _margin_rows(N, n, g, ties=False):
    """A rows whose Q argmax has a clear top-2 margin (ties: row i duplicates its max at a later column too)."""
    a = torch.rand(N, n, generator=g, dtype=torch.float64) * 0.5
    k = torch.randint(0, n, (N,), generator=g)
    a[torch.arange(N), k] += 1.0
    if ties and n > 1:
        j = torch.randint(0, n, (N,), generator=g)
        a[torch.arange(N), j] = a[torch.arange(N), k]
    return a


@pytest.mark.parametrize('N', [1, 7, 1024, 4096])
@pytest.mark.parametrize('n', [2, 18, 33, 1024])
@pytest.mark.parametrize('dueling', [False, True])
def test_act_greedy_argmax_ties_and_one_hot(N, n, dueling):
    g = torch.Generator().manual_seed(N * 7 + n)
    a = _margin_rows(N, n, g, ties=True)
    v = torch.randn(N, 1, generator=g, dtype=torch.float64) if dueling else None
    adv = a.float().cuda()
    val = v.float().cuda() if dueling else None
    act, oh, i64 = _act(adv, val, eps=0.0)
    q = odqn.combine(adv.double().cpu(), val.double().cpu() if dueling else None).numpy()
    expect = q.argmax(1)                                  # first index among ties
    assert (act == expect).all() and (i64 == expect).all()
    ref = np.zeros((N, n + 3), dtype=np.float32)
    ref[np.arange(N), expect] = 1.0
    assert (oh == ref).all()                              # the padding columns are zeroed as well


@pytest.mark.parametrize('N,n', [(1, 2), (7, 18), (4096, 18), (1024, 1024)])
def test_act_epsilon_one_replays_philox(N, n):
    g = torch.Generator().manual_seed(1)
    adv = _margin_rows(N, n, g).float().cuda()
    for ctr in (0, 5, 123456789):
        act, _, _ = _act(adv, None, eps=1.0, seed=17, counter=ctr)
        _, ra = odqn.act_draws(17, ctr, np.arange(N), n)
        assert (act == ra).all()
        assert act.min() >= 0 and act.max() < n


def test_act_schedule_reads_the_device_counter():
    from surreal_b200 import utils as U
    N, n = 4096, 6
    g = torch.Generator().manual_seed(2)
    a = _margin_rows(N, n, g)
    adv = a.float().cuda()
    for sch in (U.LinearSchedule(100, 0.1), U.PiecewiseSchedule([(0, 1.0), (10, 0.5), (30, 0.02)], outside_value=0.02)):
        pts = torch.tensor(sch.device_points(), dtype=torch.float64, device='cuda')
        for t in (0, 3, 10, 29, 50, 1000):
            act, _, _ = _act(adv, None, sched=pts, seed=9, counter=t)
            ref = odqn.act(a.numpy(), sch.value(t), 9, t)
            assert (act == ref).all(), (sch, t)


def _agent(mode, N=64, **kw):
    from surreal_b200.agent import QAgent
    lc, ec, sc = dqn_configs(**kw)
    ec.num_envs = N
    return QAgent(lc, ec, sc, 0, mode)


@pytest.mark.parametrize('mode', ['eval_deterministic', 'eval_stochastic'])
def test_agent_eval_modes(mode):
    N, n = 2048, 5
    ag = _agent(mode, N=N, n=n, dueling=True)
    x = torch.randn(N, 10, device='cuda')
    one_hot, idx = ag.act(x)
    torch.cuda.synchronize()
    adv, val = ag.model.forward_towers(x)
    q = odqn.combine(adv.double().cpu(), val.double().cpu()).numpy()
    eps = 0.0 if mode == 'eval_deterministic' else 0.05
    ref = odqn.act(q, eps, ag.seed, 0)
    got = idx.view(-1).cpu().numpy()
    top2 = np.sort(q, 1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 1e-5                # rows whose fp32 argmax cannot differ from the float64 one
    assert (got == ref)[clear].all() and clear.mean() > 0.99
    assert (one_hot.cpu().numpy().argmax(1) == got).all()
    if mode == 'eval_stochastic':
        assert 0 < (got != q.argmax(1)).sum() < N // 10
    assert ag.T == 1


def _td_case(B, n, dueling, double_q, weighted, seed=0):
    g = torch.Generator().manual_seed(seed)
    t = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    # the online rows at s' carry exact ties (the max duplicated at another column) while the target rows differ at the
    # tied columns: a double-Q argmax that did not take the first index would pick another target value
    qa, ta, oa = t(B, n) * 2, _margin_rows(B, n, g), _margin_rows(B, n, g, ties=True)
    qv, tv, ov = (t(B, 1), t(B, 1), t(B, 1)) if dueling else (None, None, None)
    actions = torch.randint(0, n, (B,), generator=g).double()
    rewards = t(B) * 2
    dones = (torch.rand(B, generator=g) < 0.2).double()
    w = torch.rand(B, generator=g, dtype=torch.float64) + 0.5 if weighted else None
    return dict(qa=qa, qv=qv, ta=ta, tv=tv, oa=oa if double_q else None, ov=ov if double_q else None, actions=actions,
                rewards=rewards, dones=dones, w=w)


def _run_td(c, B, n, gamma, eps=1e-6):
    from surreal_b200 import _lib, ops
    f = lambda x, w=None: (x.float().cuda().contiguous() if x is not None else None)  # noqa: E731
    qa, qv, ta, tv, oa, ov = (f(c[k]) for k in ('qa', 'qv', 'ta', 'tv', 'oa', 'ov'))
    act, rew, done, w = f(c['actions']), f(c['rewards']), f(c['dones']), f(c['w'])
    da = torch.full((B, ops._ru(n, 4)), 9.0, device='cuda')
    dv = torch.full((B, 4), 9.0, device='cuda') if qv is not None else None
    prio = torch.zeros(B, device='cuda')
    stats = torch.zeros(8, device='cuda')
    ws = torch.zeros(_lib.lib().sb200_dqn_workspace_bytes(B), dtype=torch.uint8, device='cuda')
    p = lambda x: C.c_void_p(x.data_ptr()) if x is not None else None  # noqa: E731
    ld = lambda x: x.stride(0) if x is not None else 0  # noqa: E731
    _lib.check(_lib.lib().sb200_dqn_td_f32(p(qa), ld(qa), p(qv), ld(qv), p(ta), ld(ta), p(tv), ld(tv), p(oa), ld(oa),
                                           p(ov), ld(ov), p(act), p(rew), p(done), p(w), B, n, gamma, eps, p(da), ld(da),
                                           p(dv), ld(dv), p(prio), p(stats), p(ws), ops._stream()), 'td')
    torch.cuda.synchronize()
    off = int(_lib.lib().sb200_dqn_bad_action_offset())
    bad = int(ws[off:off + 4].view(torch.int32).item())
    return da.cpu(), (dv.cpu() if dv is not None else None), prio.cpu(), stats.cpu(), bad


@pytest.mark.parametrize('dueling', [False, True])
@pytest.mark.parametrize('double_q', [False, True])
@pytest.mark.parametrize('weighted', [False, True])
@pytest.mark.parametrize('B,n', [(1, 2), (300, 7), (4096, 18)])
def test_td_kernel_against_float64_autograd(dueling, double_q, weighted, B, n):
    gamma = 0.97
    c = _td_case(B, n, dueling, double_q, weighted, seed=B + n)
    # the float64 reference sees the float32 inputs the kernel sees
    r = {k: (v.float().double().requires_grad_(k in ('qa', 'qv')) if v is not None else None) for k, v in c.items()}
    loss, td = odqn.td_loss(r['qa'], r['qv'], r['ta'], r['tv'], r['oa'], r['ov'], r['actions'], r['rewards'],
                            r['dones'], r['w'], gamma)
    loss.backward()
    da, dv, prio, stats, bad = _run_td(c, B, n, gamma)
    assert bad == 0
    tol = dict(rtol=1e-5, atol=2e-6 / B)                  # float32 td: a few ulp of |q| + |y|, over B
    assert torch.allclose(da[:, :n].double(), r['qa'].grad, **tol)
    assert (da[:, n:] == 0).all()
    if dueling:
        assert torch.allclose(dv[:, 0].double(), r['qv'].grad.view(-1), **tol)
        assert (dv[:, 1:] == 0).all()
    loss = float(loss.detach())
    assert abs(float(stats[0]) - loss) <= 1e-5 * max(1.0, abs(loss))
    assert abs(float(stats[1]) - float(td.abs().mean())) <= 1e-5 * max(1.0, float(td.abs().mean()))
    assert torch.allclose(prio.double(), td.detach().abs() + 1e-6, rtol=1e-5, atol=1e-6)
    assert (td.detach().abs() < 1).any() and (td.detach().abs() > 1).any() or B == 1     # both Huber branches


def test_td_kernel_flags_bad_actions_and_is_deterministic():
    B, n = 1000, 6
    c = _td_case(B, n, True, True, True, seed=5)
    first = _run_td(c, B, n, 0.99)
    again = _run_td(c, B, n, 0.99)
    assert all(torch.equal(x, y) for x, y in zip(first[:4], again[:4]))
    for badv in (-1.0, 6.0, 2.5, float('nan')):
        c2 = dict(c)
        c2['actions'] = c['actions'].clone()
        c2['actions'][17] = badv
        *_, stats, bad = _run_td(c2, B, n, 0.99)
        assert bad == 1 and float(stats[4]) == 1.0


def _learner(**kw):
    from surreal_b200.learner import DQNLearner
    lc, ec, sc = dqn_configs(**kw)
    return DQNLearner(lc, ec, sc)


def _layers(net):
    return [tuple(t.cpu() for t in net.get_layer(l)) for l in range(net.n_layers)]


def _batch(B, D, n, g, bad=False):
    b = dict(obs=torch.randn(B, D, generator=g), obs_next=torch.randn(B, D, generator=g),
             actions=torch.randint(0, n, (B, 1), generator=g).float(), rewards=torch.randn(B, 1, generator=g) * 3,
             dones=(torch.rand(B, 1, generator=g) < 0.2).float())
    return b


@pytest.mark.parametrize('dueling', [False, True])
@pytest.mark.parametrize('double_q', [False, True])
def test_learner_against_the_float64_oracle_across_target_copies(dueling, double_q):
    B, D, n, period = 64, 10, 5, 150                      # the period is not a multiple of the batch
    L = _learner(B=B, D=D, n=n, dueling=dueling, double_q=double_q, period=period, lr=3e-3, clip=1.0)
    O = odqn.OracleDQN(_layers(L.model.action_net), _layers(L.model.state_net) if dueling else None, 3e-3, 0.99,
                       double_q, period, grad_norm_clipping=1.0)
    g = torch.Generator().manual_seed(11)
    for it in range(8):
        b = _batch(B, D, n, g)
        st = L.learn({k: v.cuda() for k, v in b.items()})
        so = O.update(b['obs'], b['actions'], b['rewards'], b['obs_next'], b['dones'])
        for k in ('td_error', 'loss', 'q_value'):
            assert abs(st[k] - so[k]) <= 1e-5 * max(1.0, abs(so[k])), (it, k, st[k], so[k])
    for net, ol in [(L.model.action_net, O.a)] + ([(L.model.state_net, O.v)] if dueling else []):
        for (w, b_), (ow, ob) in zip(_layers(net), ol):
            assert torch.allclose(w.double(), ow.detach(), rtol=1e-4, atol=1e-5)
            assert torch.allclose(b_.double(), ob.detach(), rtol=1e-4, atol=1e-5)
    for (w, _), (ow, _) in zip(_layers(L.model_target.action_net), O.ta):
        assert torch.allclose(w.double(), ow, rtol=1e-4, atol=1e-5)
    assert L.target_update_samples == O.samples == 8 * B


def test_learner_rejects_bad_actions_without_changing_anything():
    B, D, n = 64, 10, 5
    L = _learner(B=B, D=D, n=n)
    g = torch.Generator().manual_seed(2)
    b = _batch(B, D, n, g)
    b['actions'][3] = n
    before = [p.clone() for net in L.model.nets() for p in (net.params,)]
    with pytest.raises(AssertionError):
        L.learn({k: v.cuda() for k, v in b.items()})
    assert all(torch.equal(x, net.params) for x, net in zip(before, L.model.nets()))


def _filled_replay(lc, ec, sc, prioritized=False, count=3000, seed=0):
    from surreal_b200.replay import UniformReplay, PrioritizedReplay
    R = (PrioritizedReplay if prioritized else UniformReplay)(lc, ec, sc)
    g = torch.Generator().manual_seed(seed)
    C_, D, n = R.memory_size, R.D, int(ec.action_spec['dim'][0])
    R.r_obs[:count] = torch.randn(count, D, generator=g).cuda()
    R.r_obs_next[:count] = torch.randn(count, D, generator=g).cuda()
    R.r_act[:count] = torch.randint(0, n, (count, 1), generator=g).float().cuda()
    R.r_rew[:count] = torch.randn(count, generator=g).cuda()
    R.r_done[:count] = (torch.rand(count, generator=g) < 0.1).float().cuda()
    R.state[0], R.state[1], R.state[3] = count % C_, count, count
    R.mark_device_inserts()
    R.snapshot_view(0)
    return R


@pytest.mark.parametrize('prioritized', [False, True])
def test_learn_from_replay_graph_equals_eager(prioritized, monkeypatch):
    out = []
    for graphs in ('1', '0'):
        monkeypatch.setenv('SB200_CUDA_GRAPH', graphs)
        torch.manual_seed(4)
        L = _learner(B=128, period=300, prioritized=prioritized)
        lc, ec, sc = dqn_configs(B=128, period=300, prioritized=prioritized)
        R = _filled_replay(lc, ec, sc, prioritized)
        L.attach_replay(R)
        sts = [L.learn_from_replay(R, K) for K in (1, 8, 8)]
        torch.cuda.synchronize()
        out.append((sts, [n.params.clone() for n in L.model.nets() + L.model_target.nets()], L.target_update_samples,
                    R.t_leaf.clone() if prioritized else None))
    (s1, p1, c1, l1), (s2, p2, c2, l2) = out
    for a, b in zip(s1, s2):
        assert {k: v for k, v in a.items() if not k.startswith('perf')} == \
            {k: v for k, v in b.items() if not k.startswith('perf')}
    assert all(torch.equal(a, b) for a, b in zip(p1, p2))
    assert c1 == c2 == 17 * 128
    if prioritized:
        assert torch.equal(l1, l2)


def test_per_priorities_are_the_td_errors_and_weights_are_used():
    B = 256
    lc, ec, sc = dqn_configs(B=B, prioritized=True)
    lc.algo.prioritized.alpha = 0.7
    torch.manual_seed(6)
    L = _learner(B=B, prioritized=True)
    R = _filled_replay(lc, ec, sc, prioritized=True)
    assert R.alpha == 0.7 and R.priority_eps == lc.algo.prioritized.eps
    R.update_priorities(np.arange(3000), np.random.default_rng(0).uniform(0.1, 5.0, 3000))    # unequal weights
    L.attach_replay(R)
    O = odqn.OracleDQN(_layers(L.model.action_net), _layers(L.model.state_net), 1e-3, 0.99, True, 100)
    b = R.sample(B)
    host = {k: (v['low_dim']['flat_inputs'] if isinstance(v, dict) else v).cpu().numpy() for k, v in b.items()}
    st = L.learn(b)
    so = O.update(host['obs'], host['actions'], host['rewards'], host['obs_next'], host['dones'], host['weights'])
    assert abs(st['loss'] - so['loss']) <= 1e-5 * max(1.0, abs(so['loss']))
    assert abs(st['avg_is_weight'] - float(host['weights'].mean())) <= 1e-6
    prio = L.td_priorities.cpu().double()
    assert torch.allclose(prio, so['td'].abs() + lc.algo.prioritized.eps, rtol=1e-4, atol=1e-6)
    leaves = torch.from_numpy(R.priorities()).double()
    idx = torch.as_tensor(b['indices']).long()
    last = {int(i): k for k, i in enumerate(idx)}                    # the last of equal indices wins
    ks = torch.tensor(list(last.values()))
    assert torch.allclose(leaves[torch.tensor(list(last.keys()))], prio[ks].float().double() ** 0.7, rtol=1e-5)
    assert not np.allclose(host['weights'], 1.0)                     # the weights are not all one: they are used


def _run_engine(overlap, prioritized=False, steps=16, watch_actor=False):
    from surreal_b200.launch import SurrealDefaultLauncher, ReplayEngine
    from surreal_b200.agent import QAgent
    from surreal_b200.learner import DQNLearner
    from surreal_b200.replay import UniformReplay, PrioritizedReplay
    from surreal_b200.main.dqn_configs import make_discrete_synthetic_env_config
    N, T, K = 32, 8, 4
    lc, ec, sc = dqn_configs(D=12, n=6, hidden=(48, 32), B=64, period=200, memory_size=2000, start=600, steps=500,
                             prioritized=prioritized)
    make_discrete_synthetic_env_config(ec, N, 12, 6, seed=1)
    ec.num_agents, ec.limit_episode_length = N, 20
    sc.agent.fetch_parameter_interval = 16
    lc.parameter_publish.min_publish_interval = 0
    torch.manual_seed(3)
    la = SurrealDefaultLauncher(QAgent, DQNLearner, PrioritizedReplay if prioritized else UniformReplay, sc, ec, lc)
    agent, replay, learner = la.setup_engine()
    eng = ReplayEngine(agent, replay, learner, T, K, overlap=overlap)
    eng.prime()
    stats, changes = [], 0
    flat = lambda m: torch.cat([n_.params for n_ in m.nets()])  # noqa: E731
    actor_prev = published = None
    for _ in range(steps):
        st = eng.step()
        if st is not None:
            stats.append([st[k] for k in ('td_error', 'loss', 'q_value')])
        if watch_actor:
            # the actors' towers change only through a parameter fetch, and only to what the learner last published
            eng.drain()
            now = flat(agent.model)
            if actor_prev is not None and not torch.equal(now, actor_prev):
                changes += 1
                assert published is not None and torch.equal(now, published)
            actor_prev = now
            if st is not None:
                published = flat(learner.model)
    eng.drain()
    if watch_actor:
        assert changes >= 2
    assert len(stats) > 0 and np.isfinite(np.array(stats)).all()
    acts = replay.r_act[:int(replay.state[1])].view(-1)
    assert (acts == acts.round()).all() and acts.min() >= 0 and acts.max() < 6
    ring = [t.clone() for t in (replay.r_obs, replay.r_obs_next, replay.r_act, replay.r_rew, replay.r_done, replay.state)]
    return ring, [n.params.clone() for n in learner.model.nets() + agent.model.nets()], stats, agent.T


@pytest.mark.parametrize('prioritized', [False, True])
def test_engine_two_streams_equal_the_one_stream_schedule(prioritized):
    r2, p2, s2, t2 = _run_engine(True, prioritized)
    r1, p1, s1, t1 = _run_engine(False, prioritized, watch_actor=True)
    assert s1 == s2 and t1 == t2 == 17 * 8
    for a, b in zip(r1 + p1, r2 + p2):
        assert torch.equal(a, b)


class _HostDiscreteEnv:
    """Batched host env: numpy observations, int actions."""

    def __init__(self, N, D, n, seed=0):
        self.N, self.D, self.A = N, D, n
        self.rng = np.random.RandomState(seed)
        self.sent = []

    def reset(self):
        self.obs = self.rng.randn(self.N, self.D).astype(np.float32)
        return {'low_dim': {'flat_inputs': self.obs}}, {}

    def step(self, action):
        a = np.asarray(action)
        assert a.dtype == np.int64 and a.shape == (self.N,)
        nxt = self.rng.randn(self.N, self.D).astype(np.float32)
        rew = self.rng.randn(self.N)
        done = np.zeros(self.N, dtype=np.float32)
        self.sent.append((self.obs.copy(), a.copy(), nxt.copy(), rew.copy()))
        self.obs = nxt
        return {'low_dim': {'flat_inputs': nxt}}, rew, done, {}


def test_host_env_loop_records_what_the_host_sent():
    from surreal_b200.agent import QAgent
    from surreal_b200.replay import UniformReplay
    N, D, n = 16, 10, 5
    lc, ec, sc = dqn_configs(D=D, n=n)
    ec.num_envs, ec.limit_episode_length = N, 6
    R = UniformReplay(lc, ec, sc)
    ag = QAgent(lc, ec, sc, 0, 'training')
    env = _HostDiscreteEnv(N, D, n)
    ag.env = w = ag.prepare_env_agent(env)
    o, _ = w.reset()
    for _ in range(6):
        o, _, _, _ = w.step(ag.act(o['low_dim']['flat_inputs']))
    torch.cuda.synchronize()
    assert len(R) == 6 * N and ag.T == 6
    for t, (o, a, on, r) in enumerate(env.sent):
        sl = slice(t * N, (t + 1) * N)
        assert np.array_equal(R.r_obs[sl].cpu().numpy(), o)
        assert np.array_equal(R.r_act[sl].view(-1).cpu().numpy(), a.astype(np.float32))
        assert np.array_equal(R.r_obs_next[sl].cpu().numpy(), on)
        assert np.allclose(R.r_rew[sl].cpu().numpy(), r.astype(np.float32))


@pytest.mark.parametrize('dueling', [False, True])
def test_checkpoint_restore_continues_bit_identically(dueling, tmp_path):
    from surreal_b200.learner import DQNLearner
    B, D, n = 64, 10, 5

    def make(folder, restore_from=None):
        lc, ec, sc = dqn_configs(B=B, D=D, n=n, dueling=dueling, period=100)
        sc.folder = str(folder)
        sc.checkpoint.learner.periodic = 1
        sc.checkpoint.learner.min_interval = 0
        sc.checkpoint.learner.include_optimizer = True
        if restore_from is not None:
            sc.checkpoint.restore = True
            sc.checkpoint.restore_folder = str(restore_from)
        return DQNLearner(lc, ec, sc)
    torch.manual_seed(1)
    A_ = make(tmp_path / 'a')
    g = torch.Generator().manual_seed(3)
    batches = [{k: v.cuda() for k, v in _batch(B, D, n, g).items()} for _ in range(4)]
    for b in batches[:3]:
        A_.learn(b)
    sd = A_.model.state_dict()
    assert list(sd)[:2] == ['fc_action_layers.0.weight', 'fc_action_layers.0.bias']
    assert any(k.startswith('fc_state_layers.') for k in sd) == dueling
    torch.manual_seed(99)                                       # the fresh learner starts from DIFFERENT weights
    B_ = make(tmp_path / 'b', restore_from=tmp_path / 'a')
    assert B_.current_iteration == 3 and B_.target_update_samples == 3 * B
    sa, sb = A_.learn(batches[3]), B_.learn(batches[3])
    torch.cuda.synchronize()
    assert {k: v for k, v in sa.items() if not k.startswith('perf')} == \
        {k: v for k, v in sb.items() if not k.startswith('perf')}
    for x, y in zip(A_.model.nets() + A_.model_target.nets(), B_.model.nets() + B_.model_target.nets()):
        assert torch.equal(x.params, y.params)


CASES = ['duel_double', 'duel_single', 'noduel_double', 'noduel_single']


def _golden_sd(g, prefix):
    return {k[len(prefix):].replace('/', '.'): torch.from_numpy(g[k]) for k in g.z.files if k.startswith(prefix)}


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('graphs', ['1', '0'])
def test_learner_against_reference_goldens(golden, case, graphs, monkeypatch):
    """DQNLearner.learn against the reference's DQNLearner (dqn_optimize_*.npz): the first update with unit weights, the
    rest with importance weights; statistics <= 1e-5, parameters and target parameters within 2e-5 (2 % of one Adam
    step at lr 1e-3) after every update, the target copies on the updates where the sample count crosses the period,
    and the priorities |td| + eps of the weighted updates."""
    monkeypatch.setenv('SB200_CUDA_GRAPH', graphs)
    g = golden('dqn_optimize_' + case)
    cfg, stats = g.js('cfg'), g.js('stats')
    from surreal_b200.learner import DQNLearner
    lc, ec, sc = dqn_configs(D=cfg['D'], n=cfg['n_actions'], hidden=cfg['hidden'], B=cfg['B'], dueling=cfg['dueling'],
                             double_q=cfg['double_q'], period=cfg['period'], lr=cfg['lr'],
                             clip=cfg['grad_norm_clipping'])
    lc.algo.gamma = cfg['gamma']
    L = DQNLearner(lc, ec, sc)
    L.model.load_state_dict(_golden_sd(g, 'init/model/'))
    L.model_target.load_state_dict(_golden_sd(g, 'init/target/'))
    eps = lc.algo.prioritized.eps
    for it in range(cfg['iters']):
        p = 'it%d/' % it
        b = {k: torch.from_numpy(g[p + k]).float().cuda() for k in ('obs', 'obs_next', 'actions', 'rewards', 'dones')}
        if it > 0:
            b['weights'] = torch.from_numpy(g[p + 'weights']).cuda()
        st = L.learn(b)
        for k in ('td_error', 'loss'):
            assert abs(st[k] - stats[it][k]) <= 1e-5 * max(1.0, abs(stats[it][k])), (case, it, k, st[k], stats[it][k])
        if it > 0:
            prio = L.td_priorities.cpu().double().numpy()
            assert np.abs(prio - (np.abs(g['td'][it]) + eps)).max() <= 1e-5, (case, it)
        for mine, net in ((L.model, 'model'), (L.model_target, 'target')):
            ref = _golden_sd(g, p + net + '/')
            for k, v in mine.state_dict().items():
                d = float((v.cpu() - ref[k]).abs().max())
                assert d <= 2e-5, (case, it, net, k, d)
    assert L.target_update_samples == cfg['iters'] * cfg['B']

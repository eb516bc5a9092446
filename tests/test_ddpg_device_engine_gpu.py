"""DDPG training on one GPU: the device sampler of UniformReplay against its CPU restatement bit for bit, K learner
updates per graph against K hand-driven ones, the stable sampling view under concurrent inserts, and ReplayEngine on two
streams against the one-stream schedule."""
import numpy as np
import pytest
import torch

from helpers import ddpg_configs
from test_uniform_device_sampler import COUNTS, device_sample_indices, sampling_view

pytestmark = pytest.mark.gpu

FIELDS = ('obs', 'obs_next', 'actions', 'rewards', 'dones')
STAT_KEYS = ('actor_loss', 'critic_loss', 'action_norm', 'rewards', 'Q_target', 'Q_policy')


def _replay(capacity, D=12, A=4, B=64, seed=0, sampler_seed=None, **cfg):
    from surreal_b200.replay import UniformReplay
    lc, ec, sc = ddpg_configs(D=D, A=A, B=B, memory_size=capacity, start=0, **cfg)
    if sampler_seed is not None:
        lc.replay.sampler_seed = sampler_seed
    r = UniformReplay(lc, ec, sc)
    g = torch.Generator(device='cuda').manual_seed(seed)
    for t in (r.r_obs, r.r_obs_next, r.r_rew):
        t.normal_(generator=g)
    r.r_act.uniform_(-1, 1, generator=g)
    r.r_done.copy_((torch.rand(capacity, generator=g, device='cuda') < 0.1).float())
    return r, (lc, ec, sc)


def _set_view(r, start, count, capacity=None):
    r.view.copy_(torch.tensor([start, count, r.memory_size if capacity is None else capacity]))


def _ring_rows(r, idx):
    return dict(obs=r.r_obs[idx], obs_next=r.r_obs_next[idx], actions=r.r_act[idx], rewards=r.r_rew[idx][:, None],
                dones=r.r_done[idx][:, None])


def _nan_out(r, B, pad=3):
    f = lambda w: torch.full((B + pad, w), float('nan'), device='cuda')  # noqa: E731
    full = dict(obs=f(r.D), obs_next=f(r.D), actions=f(r.A), rewards=f(1), dones=f(1))
    return full, {k: v[:B] for k, v in full.items()}


@pytest.mark.parametrize('count', COUNTS)
def test_sampler_matches_the_oracle_bit_for_bit(count):
    C_, B, seed, ctr = 2 ** 20 + 8, 4097, 1234567, 41
    r, _ = _replay(C_, sampler_seed=seed)
    for start in (0, C_ - 3):                                  # a view from slot 0, and one that wraps the ring's end
        _set_view(r, start, count)
        r.sampler[0] = ctr
        full, out = _nan_out(r, B)
        batch = r.sample_device(B, out=out)
        torch.cuda.synchronize()
        want = device_sample_indices(seed, ctr, start, count, C_, B)
        got = batch['indices'].cpu().numpy()
        assert np.array_equal(got, want)
        rows = _ring_rows(r, batch['indices'])
        assert torch.equal(batch['obs']['low_dim']['flat_inputs'], rows['obs'])
        assert torch.equal(batch['obs_next']['low_dim']['flat_inputs'], rows['obs_next'])
        for k in ('actions', 'rewards', 'dones'):
            assert torch.equal(batch[k], rows[k]) and batch[k].shape == rows[k].shape
        for k in FIELDS:
            assert torch.isnan(full[k][B:]).all(), 'padding rows of %s were written' % k
        assert r.draw_counter == ctr + 1 and r.sampler_status == 0
        ctr += 1


def test_sampler_on_an_empty_view_touches_nothing():
    r, _ = _replay(256)
    _set_view(r, 0, 0)
    r.sampler[0] = 9
    full, out = _nan_out(r, 64)
    idx_before = r._dev_indices.clone()
    r.sample_device(64, out=out)
    torch.cuda.synchronize()
    assert r.sampler_status == 1 and r.draw_counter == 9
    assert all(torch.isnan(v).all() for v in full.values())
    assert torch.equal(r._dev_indices, idx_before)
    _set_view(r, 0, 5)
    r.sample_device(64, out=out)
    assert r.sampler_status == 0 and r.draw_counter == 10


def test_view_kernel_follows_the_rule_over_the_wrap():
    r, _ = _replay(100)
    for reserve in (0, 30, 50):
        for total in (0, 1, 69, 70, 71, 99, 100, 101, 130, 257):
            r.state.copy_(torch.tensor([total % 100, min(total, 100), 100, total]))
            r.snapshot_view(reserve)
            start, count = sampling_view(total % 100, min(total, 100), 100, reserve)
            assert r.view.tolist() == [start, count, 100], (reserve, total)


def test_replaying_a_captured_sample_draws_fresh_indices():
    from surreal_b200 import _lib
    r, _ = _replay(5000, B=64, sampler_seed=77)
    _set_view(r, 4990, 3000)
    c = 5
    r.sampler[0] = c
    _, out = _nan_out(r, 64, pad=0)
    _lib.ensure_device()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        batch = r.sample_device(64, out=out)
    seen = []
    for k in range(3):
        g.replay()
        torch.cuda.synchronize()
        got = batch['indices'].cpu().numpy()
        assert np.array_equal(got, device_sample_indices(77, c + k, 4990, 3000, 5000, 64))
        assert torch.equal(batch['actions'], r.r_act[batch['indices']])
        seen.append(got.tolist())
    assert seen[0] != seen[1] != seen[2] != seen[0]
    assert r.draw_counter == c + 3


# ---- learner ----------------------------------------------------------------------------------------------------
def _learner_state(L):
    ts = [L.model.actor.params, L.model.critic.params, L.model_target.actor.params, L.model_target.critic.params]
    opts = [L.actor_optim, L.critic_optim]
    if L.use_double_critic:
        ts += [L.model2.critic.params, L.model_target2.critic.params]
        opts.append(L.critic_optim2)
    for o in opts:
        ts += [o.exp_avg, o.exp_avg_sq]
    return [t.clone() for t in ts]


def _twin(target, graphs=True, layernorm=False, td3=False):
    """(replay, learner A, learner B): two learners from one seed over one ring."""
    from surreal_b200.learner import DDPGLearner
    r, _ = _replay(600, D=9, A=3, B=16, sampler_seed=3)
    _set_view(r, 590, 500)
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
    for call in range(2):                                      # the second call replays the captured graph
        c = r.draw_counter
        sa = LA.learn_from_replay(r, updates=K)
        r.sampler[0] = c
        for _ in range(K):
            sb = LB.learn(r.sample_device(16, out=LB.replay_out_buffers()))
        torch.cuda.synchronize()
        assert r.draw_counter == c + K
        for a, b in zip(_learner_state(LA), _learner_state(LB)):
            assert torch.equal(a, b)
        for k in STAT_KEYS + (('Q_policy2',) if case == 'td3' else ()):
            assert sa[k] == sb[k], k
        assert LA.current_iteration == LB.current_iteration == K * (call + 1)
        if target['type'] == 'hard':
            assert LA.target_update_counter == LB.target_update_counter == K * (call + 1)
    if target['type'] == 'hard':                               # 10 updates, interval 3: the last copy was at update 9
        assert not torch.equal(LA.model_target.critic.params, LA.model.critic.params)


def test_bad_action_in_a_sampled_record_leaves_the_learner_untouched():
    r, LA, _ = _twin({'type': 'soft', 'tau': 0.01, 'interval': 1})
    LA.learn_from_replay(r, updates=3)                         # good batches first (captures the graph, moves Adam)
    snap = _learner_state(LA)
    r.r_act[7, 1] = 1.5
    _set_view(r, 7, 1)                                         # every draw is the bad record
    with pytest.raises(AssertionError):
        LA.learn_from_replay(r, updates=3)
    torch.cuda.synchronize()
    for a, b in zip(snap, _learner_state(LA)):
        assert torch.equal(a, b)
    r.r_act[7, 1] = 0.5
    st = LA.learn_from_replay(r, updates=3)                    # and the learner goes on afterwards
    assert np.isfinite(st['critic_loss']) and not torch.equal(snap[0], LA.model.actor.params)


# ---- the view under concurrent inserts ----------------------------------------------------------------------------
class _SequenceEnv:
    """Device 'env' whose k-th emitted record carries k in obs[0], obs_next[0] and the reward (the test puts it in
    action[0] too): actor i's record of step t is insert t * N + i."""
    graph_safe = True

    def __init__(self, N, D, A):
        self.N, self.D, self.A, self.device = N, D, A, torch.device('cuda', torch.cuda.current_device())
        self.t = 0
        self.ar = torch.arange(N, dtype=torch.float32, device=self.device)
        z = lambda *s: torch.zeros(*s, device=self.device)  # noqa: E731
        self.obs, self.obs_next, self.reward, self.done = z(N, D), z(N, D), z(N), z(N)

    def reset(self):
        self.obs[:, 0] = self.ar
        return {'low_dim': {'flat_inputs': self.obs}}, {}

    def step(self, action):
        seq = self.ar + float(self.t * self.N)
        self.obs_next[:, 0] = seq
        self.reward.copy_(seq)
        self.t += 1
        self.obs[:, 0] = seq + float(self.N)
        return {'low_dim': {'flat_inputs': self.obs}}, self.reward, self.done, {'obs_next': self.obs_next}


def test_no_torn_records_while_the_next_chunk_wraps_the_ring():
    from surreal_b200.env import ExpSenderWrapperSSARNStepBootstrap
    N, D, A, T, C_ = 64, 12, 4, 8, 4096
    r, (lc, ec, sc) = _replay(C_, D=D, A=A, n_step=1)
    env = ExpSenderWrapperSSARNStepBootstrap(_SequenceEnv(N, D, A), lc, sc, replay=r)
    env.reset()
    act = torch.zeros(N, A, device='cuda')

    def chunk(steps):
        for _ in range(steps):
            act[:, 0] = env.env.ar + float(env.env.t * N)
            env.step(act)

    chunk(60)                                                  # 3840 records: the next chunk of 512 wraps the ring
    W = N * T
    r.snapshot_view(reserve=W)
    torch.cuda.synchronize()
    start, count, cap = r.view.tolist()
    assert (start, count, cap) == (sampling_view(3840, 3840, C_, W) + (C_,)) and start == 256
    sA, sL = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [_nan_out(r, 4096, pad=0)[1] for _ in range(8)]
    idxs = []
    with torch.cuda.stream(sA):
        chunk(T)
    with torch.cuda.stream(sL):
        for o in outs:
            idxs.append(r.sample_device(4096, out=o)['indices'].clone())
    torch.cuda.synchronize()
    assert r.state.tolist() == [(3840 + W) % C_, C_, C_, 3840 + W]
    for o, idx in zip(outs, idxs):
        seq = o['rewards'][:, 0]
        assert torch.equal(o['obs'][:, 0], seq) and torch.equal(o['obs_next'][:, 0], seq)
        assert torch.equal(o['actions'][:, 0], seq)
        assert torch.equal(seq.long() % C_, idx)               # the record that slot held at the snapshot
        assert bool((((idx - start) % C_) < count).all()) and float(seq.max()) < 3840


# ---- engine -------------------------------------------------------------------------------------------------------
def _emitted(steps, episode=20, n_step=3):
    """Records one actor has emitted after ``steps`` env steps: from the n_step-th step of every episode on."""
    return steps // episode * (episode - n_step + 1) + max(0, steps % episode - (n_step - 1))


def _run_engine(overlap, steps=20, watch_actor=False):
    from surreal_b200.launch import SurrealDefaultLauncher, ReplayEngine
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.learner import DDPGLearner
    from surreal_b200.replay import UniformReplay
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    N, T, K = 32, 8, 4
    lc, ec, sc = ddpg_configs(D=12, A=4, actor_h=(48, 32), critic_h=(64, 48), B=64, n_step=3, memory_size=2000,
                              start=1000, target={'type': 'hard', 'interval': 7})
    make_synthetic_env_config(ec, N, 12, 4, seed=1)
    ec.num_agents = N
    ec.limit_episode_length = 20
    sc.agent.fetch_parameter_interval = 16                     # a fetch every second chunk
    lc.parameter_publish.min_publish_interval = 0              # a publish after every learner step
    torch.manual_seed(3)
    la = SurrealDefaultLauncher(DDPGAgent, DDPGLearner, UniformReplay, sc, ec, lc)
    agent, replay, learner = la.setup_engine()
    eng = ReplayEngine(agent, replay, learner, T, K, overlap=overlap)
    eng.prime()
    stats, idle, changes = [], 0, 0
    actor_prev = published = None
    for j in range(steps):
        st = eng.step()
        if st is None:
            idle += 1
            assert learner.current_iteration == 0              # the learner waits for size > sampling_start_size
        else:
            stats.append([st[k] for k in STAT_KEYS])
        if watch_actor:
            eng.drain()
            now = agent.model.actor.params.clone()
            if actor_prev is not None and not torch.equal(now, actor_prev):
                changes += 1                                   # only ever to what the learner last published
                assert published is not None and torch.equal(now, published)
            actor_prev = now
            if st is not None:
                published = learner.model.actor.params.clone()
    eng.drain()
    assert idle == next(c for c in range(1, 99) if N * _emitted(T * c) > 1000) - 1
    assert learner.current_iteration == K * (steps - idle)
    assert int(replay.state[3]) == N * _emitted(T * (steps + 1))
    assert np.isfinite(np.array(stats)).all()
    if watch_actor:
        assert changes >= 2
    ring = [t.clone() for t in (replay.r_obs, replay.r_obs_next, replay.r_act, replay.r_rew, replay.r_done, replay.state)]
    return ring, _learner_state(learner) + [agent.model.actor.params.clone()], stats


def test_engine_two_streams_equal_the_one_stream_schedule():
    ring2, params2, stats2 = _run_engine(overlap=True)
    ring1, params1, stats1 = _run_engine(overlap=False, watch_actor=True)
    assert stats1 == stats2
    for a, b in zip(ring1 + params1, ring2 + params2):
        assert torch.equal(a, b)


def test_engine_rejects_a_ring_smaller_than_two_chunks():
    from surreal_b200.launch import SurrealDefaultLauncher, ReplayEngine
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.learner import DDPGLearner
    from surreal_b200.replay import UniformReplay
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    from surreal_b200.session import ConfigError
    lc, ec, sc = ddpg_configs(D=12, A=4, B=64, memory_size=500, start=10)
    make_synthetic_env_config(ec, 32, 12, 4, seed=1)
    ec.num_agents = 32
    agent, replay, learner = SurrealDefaultLauncher(DDPGAgent, DDPGLearner, UniformReplay, sc, ec, lc).setup_engine()
    with pytest.raises(ConfigError):
        ReplayEngine(agent, replay, learner, 8, 4)             # 2 x 32 x 8 = 512 > 500


def test_ddpg_launcher_trains_and_returns(tmp_path):
    import os
    from surreal_b200.main.ddpg_configs import DDPGLauncher
    la = DDPGLauncher()
    learner = la.main(['learner', '--', '--env', 'synthetic:12:4', '--num-agents', '32', '--experiment-folder',
                       str(tmp_path), '--unit-test', '--rollout-steps', '8', '--updates-per-chunk', '2',
                       '--iterations', '4'])
    assert os.path.exists(os.path.join(str(tmp_path), 'config.yml'))
    assert learner.current_iteration == 2 * 4                  # 32 x 6 records after the first chunk > 5: no idle step
    assert int(la.replay.state[3]) > 0

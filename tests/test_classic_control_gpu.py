"""The classic-control tasks on the device (csrc/env.cu, surreal_b200.env.classic):

1. kernels against the float64 statement of tests/classic_ref.py: one step from random states and actions at several
   actor counts, the termination boundaries, the reset draws bit for bit, episode counters and caps at staggered
   episode ends, the fused window step against step + ppo_window_step, graph replay against eager;
2. learning: each algorithm family trains a task from a fixed seed (configs: tests/classic_learning.py) and its trained
   policy clears the bar, the untrained one does not;
3. determinism: a short run repeated at the same seed gives bit-identical parameters."""
import math

import numpy as np
import pytest
import torch

import classic_ref as cr
from helpers import ppo_configs

pytestmark = pytest.mark.gpu
DEV = 'cuda'

# float32 against float64 on one step: the kernels round every operation once and use the device's sinf / cosf (a few
# ulp); the worst error of a component is a few ulp of the largest term that enters it
STATE_TOL = 8e-6          # relative to max(1, |value|)
REWARD_TOL = 1e-5         # relative to max(1, |reward|)


def _envs():
    from surreal_b200.env import CartPoleEnv, PendulumEnv
    return {cr.CARTPOLE: CartPoleEnv, cr.PENDULUM: PendulumEnv}


def _close(got, ref, tol, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    if got.size == 0:
        return
    err = np.abs(got - ref) / np.maximum(1.0, np.abs(ref))
    assert float(err.max()) <= tol, '%s: worst relative error %.3g at %s' % (what, float(err.max()), np.argmax(err))


def _random_states(task, N, rng):
    if task == cr.CARTPOLE:
        lo, hi = np.array([-2.4, -3.0, -0.21, -3.5]), np.array([2.4, 3.0, 0.21, 3.5])
    else:
        lo, hi = np.array([-4 * math.pi, -8.0]), np.array([4 * math.pi, 8.0])
    return rng.uniform(lo, hi, (N, len(lo))).astype(np.float32)


def _random_actions(task, N, rng):
    if task == cr.CARTPOLE:
        return np.eye(2, dtype=np.float32)[rng.randint(0, 2, N)]
    return rng.uniform(-1.5, 1.5, (N, 1)).astype(np.float32)          # beyond [-1, 1]: the clip is exercised


def _near_boundary(task, nxt):
    """Successors within 1e-5 of a termination threshold, where float32 and float64 may disagree on done."""
    if task != cr.CARTPOLE:
        return np.zeros(len(nxt), dtype=bool)
    return (np.abs(np.abs(nxt[:, 0]) - cr.X_THRESHOLD) < 1e-5) | (np.abs(np.abs(nxt[:, 2]) - cr.THETA_THRESHOLD) < 1e-5)


def _set(env, state, ep_step=None, episode=None):
    env.state.copy_(torch.tensor(state, device=DEV))
    if ep_step is not None:
        env.ep_step.copy_(torch.tensor(ep_step, dtype=torch.int32, device=DEV))
    if episode is not None:
        env.episode.copy_(torch.tensor(episode, dtype=torch.int32, device=DEV))


# -- 1. kernels --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('task', [cr.CARTPOLE, cr.PENDULUM])
@pytest.mark.parametrize('N', [1, 33, 1024, 65536])
def test_one_step_matches_the_oracle(task, N):
    """Random states (CartPole: inside and around its bounds; Pendulum: several turns, every speed) and actions (Pendulum:
    beyond [-1, 1]).  Successors within 1e-5 of a termination threshold are redrawn: there float32 and float64 may
    disagree on done, and test_cartpole_boundaries_on_the_device covers them."""
    rng = np.random.RandomState(N + 7 * task)
    s = _random_states(task, N, rng)
    a = _random_actions(task, N, rng)
    while True:
        nxt, rew, term = cr.physics_step(task, s.astype(np.float64), a)
        near = _near_boundary(task, nxt)
        if not near.any():
            break
        s[near] = _random_states(task, int(near.sum()), rng)
    env = _envs()[task](N, limit_episode_length=0, seed=3 + N)
    env.reset()
    episode = rng.randint(0, 1000, N)
    _set(env, s, np.zeros(N), episode)
    obs, r, d, info = env.step(torch.tensor(a, device=DEV))
    torch.cuda.synchronize()
    _close(info['obs_next'].cpu().numpy(), cr.observe(task, nxt), STATE_TOL, 'obs_next')
    _close(r.cpu().numpy(), rew, REWARD_TOL, 'reward')
    assert np.array_equal(d.cpu().numpy(), term.astype(np.float32))
    st = env.state.cpu().numpy()
    live = ~term
    _close(st[live], nxt[live], STATE_TOL, 'state')
    assert np.array_equal(obs['low_dim']['flat_inputs'].cpu().numpy()[live],
                          info['obs_next'].cpu().numpy()[live])
    ids = np.nonzero(term)[0]
    if len(ids):                                       # terminal actors restart with their next episode index
        assert np.array_equal(st[ids], cr.reset_state(task, env.seed, episode[ids] + 1, ids))
    assert np.array_equal(env.episode.cpu().numpy(), episode + term)
    assert np.array_equal(env.ep_step.cpu().numpy(), np.where(term, 0, 1))
    if task == cr.CARTPOLE and N > 1000:
        assert 0.05 < term.mean() < 0.95                # both outcomes occur
        assert np.array_equal(r.cpu().numpy(), np.ones(N, np.float32))


def test_hand_checks_on_the_device():
    from surreal_b200.env import CartPoleEnv, PendulumEnv
    cp = CartPoleEnv(1)
    cp.reset()
    _set(cp, np.zeros((1, 4), np.float32))
    _, r, d, info = cp.step(torch.tensor([[0.0, 1.0]], device=DEV))
    np.testing.assert_allclose(info['obs_next'].cpu().numpy()[0],
                               [0.0, 0.19512195, 0.0, -0.29268293], rtol=0, atol=2e-7)
    assert float(r) == 1.0 and float(d) == 0.0
    pe = PendulumEnv(1)
    pe.reset()
    _set(pe, np.zeros((1, 2), np.float32))
    _, r, d, info = pe.step(torch.tensor([[1.0]], device=DEV))
    np.testing.assert_allclose(info['obs_next'].cpu().numpy()[0],
                               [0.99988750, 0.01499944, 0.3], rtol=0, atol=2e-7)
    assert abs(float(r) + 0.004) < 1e-9 and float(d) == 0.0


@pytest.mark.parametrize('which', [0, 2])
def test_cartpole_boundaries_on_the_device(which):
    """Successors exactly on a threshold (zero velocities keep x and theta in place) are not terminal, one float32
    beyond is, on both sides."""
    from surreal_b200.env import CartPoleEnv
    thr = cr.X_THRESHOLD if which == 0 else cr.THETA_THRESHOLD
    rows, expect = [], []
    for sign in (1.0, -1.0):
        edge = np.float32(sign * thr)
        for v, t in ((edge, False), (np.nextafter(edge, np.float32(sign * np.inf)), True),
                     (np.nextafter(edge, np.float32(0.0)), False)):
            s = np.zeros(4, np.float32)
            s[which] = v
            rows.append(s)
            expect.append(t)
    env = CartPoleEnv(len(rows))
    env.reset()
    _set(env, np.stack(rows))
    _, _, d, info = env.step(torch.tensor(np.tile([[1.0, 0.0]], (len(rows), 1)).astype(np.float32), device=DEV))
    nxt = info['obs_next'].cpu().numpy()
    assert np.array_equal(nxt[:, which], np.stack(rows)[:, which])
    assert list(d.cpu().numpy()) == [1.0 if t else 0.0 for t in expect]


@pytest.mark.parametrize('task', [cr.CARTPOLE, cr.PENDULUM])
def test_reset_draws_are_the_oracle_philox(task):
    N, seed = 5000, 77
    env = _envs()[task](N, seed=seed)
    obs, _ = env.reset()
    st = env.state.cpu().numpy()
    assert np.array_equal(st, cr.reset_state(task, seed, 0, np.arange(N)))
    o = obs['low_dim']['flat_inputs'].cpu().numpy()
    if task == cr.CARTPOLE:
        assert np.array_equal(o, st)
    else:
        _close(o, cr.observe(task, st), 2e-7, 'reset obs')
    assert not env.ep_step.any() and not env.episode.any()
    # a cap of one step: every step restarts every actor, with episode index 1, 2, ...
    env = _envs()[task](N, limit_episode_length=1, seed=seed)
    env.reset()
    a = torch.tensor(_random_actions(task, N, np.random.RandomState(0)), device=DEV)
    for k in (1, 2, 3):
        _, _, d, _ = env.step(a)
        assert bool((d == 1).all())
        assert np.array_equal(env.state.cpu().numpy(), cr.reset_state(task, seed, k, np.arange(N)))
        assert bool((env.episode == k).all()) and not env.ep_step.any()


@pytest.mark.parametrize('task', [cr.CARTPOLE, cr.PENDULUM])
def test_staggered_episode_ends(task):
    """Every actor starts at another episode step under a cap of 7: done, episode index, episode step, obs and obs_next
    against the oracle step by step, from the device's own state each step."""
    N, L, T, seed = 300, 7, 30, 5
    env = _envs()[task](N, limit_episode_length=L, seed=seed)
    env.reset()
    ep0 = np.arange(N) % L
    env.ep_step.copy_(torch.tensor(ep0, dtype=torch.int32, device=DEV))
    rng = np.random.RandomState(1)
    ep_step, episode = ep0.copy(), np.zeros(N, np.int64)
    n_done = n_term = 0
    for t in range(T):
        s = env.state.cpu().numpy()
        a = _random_actions(task, N, rng)
        nxt, rew, term = cr.physics_step(task, s.astype(np.float64), a)
        obs, r, d, info = env.step(torch.tensor(a, device=DEV))
        ep_step += 1
        ok = ~_near_boundary(task, nxt)
        done = term | (ep_step >= L)
        dv = d.cpu().numpy()
        assert np.array_equal(dv[ok], done[ok].astype(np.float32)), t
        done = dv > 0.5
        episode += done
        ep_step[done] = 0
        assert np.array_equal(env.episode.cpu().numpy(), episode) and np.array_equal(env.ep_step.cpu().numpy(), ep_step)
        on = info['obs_next'].cpu().numpy()
        o = obs['low_dim']['flat_inputs'].cpu().numpy()
        _close(on, cr.observe(task, nxt), STATE_TOL, 'obs_next')
        _close(r.cpu().numpy(), rew, REWARD_TOL, 'reward')
        assert np.array_equal(o[~done], on[~done])
        ids = np.nonzero(done)[0]
        st = env.state.cpu().numpy()
        assert np.array_equal(st[ids], cr.reset_state(task, seed, episode[ids], ids))
        _close(o[ids], cr.observe(task, st[ids]), 2e-7, 'reset obs')
        n_done += len(ids)
        n_term += int((term & done).sum())
    assert n_done >= N * T // L - N
    if task == cr.CARTPOLE:
        assert n_term == 0 or n_term < n_done                # the cap ends most episodes at L = 7


def _window_run(task, fuse, T=45):
    from surreal_b200.agent import PPOAgent
    from surreal_b200.replay import FIFOReplay
    N = 70
    D, A = (4, 2) if task == cr.CARTPOLE else (3, 1)
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=(32, 24), critic_h=(32, 24), n_step=6, stride=4, B=8, memory_size=N + 40)
    ec.num_envs = N
    if task == cr.CARTPOLE:
        ec.action_spec = {'dim': (2,), 'type': 'discrete'}
    R = FIFOReplay(lc, ec, sc)
    ag = PPOAgent(lc, ec, sc, 1, 'training')
    torch.manual_seed(5)
    ag.model.actor.params.copy_(torch.randn_like(ag.model.actor.params) * 0.3)
    ag.set_noise(np.linspace(-0.2, 0.2, N))
    # a cap of 14 = 6 + 2 x 4: a full episode's third window ends with its done
    env = _envs()[task](N, limit_episode_length=14, seed=4)
    ag.env = w = ag.prepare_env_agent(env)
    w.fuse_launches = fuse
    obs, _ = w.reset()
    env.ep_step.copy_(torch.arange(N, dtype=torch.int32, device=DEV) % 14)
    for _ in range(T):
        obs, _, _, _ = w.step(ag.act(obs))
    torch.cuda.synchronize()
    return dict(state=R._read_state(), pos=w.stage_pos.clone(), so=w.stage_obs.clone(), sa=w.stage_act.clone(),
                r_obs=R.r_obs.clone(), r_act=R.r_act.clone(), r_pd=R.r_pd.clone(), r_rew=R.r_rew.clone(),
                r_done=R.r_done.clone(), env=env.state.clone(), episode=env.episode.clone())


@pytest.mark.parametrize('task', [cr.CARTPOLE, cr.PENDULUM])
def test_fused_window_step_equals_step_and_window_commit(task):
    f, u = _window_run(task, True), _window_run(task, False)
    assert f['state'] == u['state'] and f['state']['total_in'] > 0
    for k in ('pos', 'so', 'sa', 'r_obs', 'r_act', 'r_pd', 'r_rew', 'r_done', 'env', 'episode'):
        assert torch.equal(f[k], u[k]), k
    assert int(f['episode'].sum()) > 0 and float(f['r_done'].sum()) > 0


@pytest.mark.parametrize('task', [cr.CARTPOLE, cr.PENDULUM])
def test_graph_replay_equals_eager(task):
    N, T = 513, 25
    rng = np.random.RandomState(2)
    acts = [torch.tensor(_random_actions(task, N, rng), device=DEV) for _ in range(T)]
    out = []
    for graph in (False, True):
        env = _envs()[task](N, limit_episode_length=9, seed=8)
        env.reset()
        rows = []

        def body():
            for a in acts:
                _, r, d, info = env.step(a)
                rows.append(torch.cat([info['obs_next'], env.obs, r[:, None], d[:, None]], 1))
        if graph:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                with torch.cuda.graph(g):
                    body()
            torch.cuda.current_stream().wait_stream(s)
            env.reset()                                      # capture ran no kernels: start over from the reset state
            g.replay()
        else:
            body()
        torch.cuda.synchronize()
        out.append((torch.stack(rows), env.state.clone(), env.episode.clone(), env.ep_step.clone()))
    for a, b in zip(*out):
        assert torch.equal(a, b)
    assert int(out[0][2].sum()) > 0


# -- 2. learning -------------------------------------------------------------------------------------------------------
# Budget of engine steps per case (seed 0).  The policy is evaluated every CHECK_EVERY steps; the test passes at the
# first evaluation that clears the bar.  Evaluating does not change the run (no publish), so the run is deterministic.
LEARN_BUDGET = {'ppo_cartpole_mlp': 1500, 'ppo_cartpole_default': 1500, 'dqn_cartpole': 1500, 'ddpg_pendulum': 600,
                'ppo_pendulum': 900}
CHECK_EVERY = 20


@pytest.mark.parametrize('name', list(LEARN_BUDGET))
def test_learns_the_task(name):
    import classic_learning as CL
    case = CL.CASES[name]
    run = CL.Run(case, seed=0)
    before, _ = run.evaluate()
    assert before < case.random_below, (name, 'untrained', before)
    curve = []
    for it in range(1, LEARN_BUDGET[name] + 1):
        run.step()
        if it % CHECK_EVERY == 0:
            after, rets = run.evaluate()
            curve.append(round(after, 1))
            if after >= case.bar:
                return
    raise AssertionError('%s: no evaluation reached %s in %d steps: %s' % (name, case.bar, LEARN_BUDGET[name], curve))


# -- 3. determinism ----------------------------------------------------------------------------------------------------
def _params(run):
    return [v.clone() for v in run.learner.model.state_dict().values() if isinstance(v, torch.Tensor)]


@pytest.mark.parametrize('name,iterations', [('ppo_cartpole_mlp', 3), ('ppo_cartpole_default', 8), ('dqn_cartpole', 40),
                                             ('ddpg_pendulum', 12)])
def test_same_seed_gives_bit_identical_parameters(name, iterations):
    import classic_learning as CL
    out = []
    for _ in range(2):
        run = CL.Run(CL.CASES[name], seed=3)
        for _ in range(iterations):
            run.step()
        run.sync()
        out.append(_params(run))
    assert len(out[0]) > 0
    for a, b in zip(*out):
        assert torch.equal(a, b)

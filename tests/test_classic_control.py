"""CPU checks of the classic-control tasks: the float64 statement (tests/classic_ref.py) against the hand checks, the
strict termination boundaries, the angle normalisation at +-pi, the episode cap and auto-reset; the env-name routing of
the configs, launchers and agents; the sm_90a cross-compile of csrc/env.cu."""
import copy
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import classic_ref as cr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# -- the tasks ---------------------------------------------------------------------------------------------------------
def test_cartpole_hand_check():
    nxt, rew, term = cr.cartpole_step(np.zeros((1, 4)), [True])
    assert nxt[0, 0] == 0.0 and nxt[0, 2] == 0.0
    assert abs(nxt[0, 1] - 0.19512195) < 1e-8 and abs(nxt[0, 3] - (-0.29268293)) < 1e-8
    assert rew[0] == 1.0 and not term[0]
    left, _, _ = cr.cartpole_step(np.zeros((1, 4)), [False])
    np.testing.assert_allclose(left, -nxt, rtol=0, atol=1e-15)          # the mirror image
    # both action forms of the device env: int indices and one-hot rows
    assert list(cr.push_right(np.array([1, 0]), 2)) == [True, False]
    assert list(cr.push_right(np.array([[0., 1.], [1., 0.]]), 2)) == [True, False]


def test_pendulum_hand_check():
    nxt, rew, term = cr.pendulum_step(np.zeros((1, 2)), [1.0])
    assert abs(rew[0] - (-0.004)) < 1e-15 and not term[0]
    assert abs(nxt[0, 1] - 0.3) < 1e-15 and abs(nxt[0, 0] - 0.015) < 1e-15
    np.testing.assert_allclose(cr.observe(cr.PENDULUM, nxt)[0], [0.99988750, 0.01499944, 0.3], rtol=0, atol=5e-9)
    # the action is clipped to [-1, 1] before it is scaled to the torque, and the speed to [-8, 8] before theta moves
    nxt2, rew2, _ = cr.pendulum_step(np.zeros((1, 2)), [7.5])
    assert np.array_equal(nxt2, nxt) and rew2[0] == rew[0]
    fast, _, _ = cr.pendulum_step(np.array([[math.pi / 2, 7.9]]), [1.0])
    assert fast[0, 1] == 8.0 and abs(fast[0, 0] - (math.pi / 2 + 8.0 * 0.05)) < 1e-15


@pytest.mark.parametrize('which', ['x', 'theta'])
def test_cartpole_termination_is_strict(which):
    """A state exactly on a threshold is not terminal; the next float32 beyond it is.  With zero velocities the Euler
    step leaves x and theta where they are, so the successor sits exactly on the boundary."""
    k, thr = (0, cr.X_THRESHOLD) if which == 'x' else (2, cr.THETA_THRESHOLD)
    for sign in (1.0, -1.0):
        s = np.zeros((3, 4), dtype=np.float32)
        edge = np.float32(sign * thr)
        s[0, k] = edge
        s[1, k] = np.nextafter(edge, np.float32(sign * np.inf))
        s[2, k] = np.nextafter(edge, np.float32(0.0))
        nxt, _, term = cr.cartpole_step(s.astype(np.float64), [True, True, True])
        assert list(nxt[:, k]) == list(s[:, k].astype(np.float64))
        assert list(term) == [False, True, False]
    assert cr.X_THRESHOLD == float(np.float32(2.4)) and cr.THETA_THRESHOLD == float(np.float32(12 * 2 * math.pi / 360))


def test_angle_normalize_at_pi():
    for x in (math.pi, -math.pi, 3 * math.pi, -3 * math.pi):
        assert abs(cr.angle_normalize(x) - (-math.pi)) < 1e-12
    assert cr.angle_normalize(0.0) == 0.0
    assert abs(cr.angle_normalize(2 * math.pi + 0.25) - 0.25) < 1e-12
    assert abs(cr.angle_normalize(-0.25) - (-0.25)) < 1e-15
    # the reward at theta = +-pi: the largest angle cost, pi^2, on either side
    _, r, _ = cr.pendulum_step(np.array([[math.pi, 0.0], [-math.pi, 0.0]]), [0.0, 0.0])
    np.testing.assert_allclose(r, [-math.pi ** 2, -math.pi ** 2], rtol=1e-15)


def test_reset_draws_ranges_and_keys():
    ids = np.arange(4096)
    cp = cr.reset_state(cr.CARTPOLE, 5, 0, ids)
    assert cp.dtype == np.float32 and cp.shape == (4096, 4)
    assert cp.min() >= -0.05 and cp.max() <= 0.05 and abs(float(cp.mean())) < 2e-3
    pe = cr.reset_state(cr.PENDULUM, 5, 0, ids)
    assert pe.shape == (4096, 2) and np.abs(pe[:, 0]).max() <= np.float32(math.pi) and np.abs(pe[:, 1]).max() <= 1.0
    assert np.abs(pe[:, 0]).max() > 3.0                                  # the whole circle
    # another seed, episode or actor: another draw; the same key: the same draw
    assert not np.array_equal(cp, cr.reset_state(cr.CARTPOLE, 6, 0, ids))
    assert not np.array_equal(cp, cr.reset_state(cr.CARTPOLE, 5, 1, ids))
    assert np.array_equal(cp[7:9], cr.reset_state(cr.CARTPOLE, 5, 0, [7, 8]))
    u = cr.reset_uniforms(5, 0, ids)
    assert u.dtype == np.float32 and u.min() >= 0.0 and u.max() < 1.0


def test_cap_and_auto_reset():
    """Pendulum never terminates: the cap alone ends its episodes; every done actor restarts with its next episode
    index, and obs_next keeps the true successor."""
    env = cr.ClassicRef(cr.PENDULUM, 5, limit_episode_length=3, seed=11)
    obs, _ = env.reset()
    np.testing.assert_array_equal(obs['low_dim']['flat_inputs'],
                                  cr.observe(cr.PENDULUM, cr.reset_state(cr.PENDULUM, 11, 0, np.arange(5))).astype(np.float32))
    rng = np.random.RandomState(0)
    for t in range(1, 8):
        s0 = env.state.copy()
        a = rng.uniform(-1, 1, (5, 1))
        o, r, d, info = env.step(a)
        nxt, rew, _ = cr.pendulum_step(s0, a)
        np.testing.assert_array_equal(info['obs_next'], cr.observe(cr.PENDULUM, nxt).astype(np.float32))
        np.testing.assert_array_equal(r, rew.astype(np.float32))
        assert list(d) == [1.0 if t % 3 == 0 else 0.0] * 5
        assert list(env.episode) == [t // 3] * 5
        if t % 3 == 0:
            np.testing.assert_array_equal(env.state, cr.reset_state(cr.PENDULUM, 11, t // 3, np.arange(5)))
        else:
            np.testing.assert_array_equal(o['low_dim']['flat_inputs'], info['obs_next'])
    # limit 0: the registered limit; CartPole ends an episode at the boundary as well
    assert cr.ClassicRef(cr.CARTPOLE, 2).max_steps == 500 and cr.ClassicRef(cr.PENDULUM, 2, 0).max_steps == 200
    env = cr.ClassicRef(cr.CARTPOLE, 2, seed=3)
    env.reset()
    env.state[0] = [2.39, 1.0, 0.0, 0.0]
    _, r, d, info = env.step(np.array([1, 1]))
    assert list(d) == [1.0, 0.0] and list(r) == [1.0, 1.0] and list(env.episode) == [1, 0] and list(env.ep_step) == [0, 1]
    assert info['obs_next'][0, 0] > cr.X_THRESHOLD
    np.testing.assert_array_equal(env.state[0], cr.reset_state(cr.CARTPOLE, 3, 1, [0])[0])


# -- configs and routing -----------------------------------------------------------------------------------------------
def _fresh(tree):
    from surreal_b200.session import Config
    return Config(copy.deepcopy(tree.to_dict()))


def test_make_classic_env_config():
    from surreal_b200.main.ppo_configs import PPO_DEFAULT_ENV_CONFIG, make_classic_env_config
    ec = make_classic_env_config(_fresh(PPO_DEFAULT_ENV_CONFIG), 'classic:CartPole-v1', 16, seed=4)
    assert ec.env_name == 'classic:CartPole-v1' and ec.num_envs == 16 and ec.seed == 4
    assert tuple(ec.obs_spec['low_dim']['flat_inputs']) == (4,)
    assert tuple(ec.action_spec['dim']) == (2,) and ec.action_spec['type'] == 'discrete'
    assert ec.limit_episode_length == 500
    ec = make_classic_env_config(_fresh(PPO_DEFAULT_ENV_CONFIG), 'classic:Pendulum-v1', 8)
    assert tuple(ec.obs_spec['low_dim']['flat_inputs']) == (3,)
    assert tuple(ec.action_spec['dim']) == (1,) and ec.action_spec['type'] == 'continuous'
    assert ec.limit_episode_length == 200
    for bad in ('classic:Acrobot-v1', 'synthetic', 'CartPole-v1'):
        with pytest.raises(ValueError):
            make_classic_env_config(_fresh(PPO_DEFAULT_ENV_CONFIG), bad, 8)


@pytest.mark.parametrize('launcher,name,kind,D,A', [
    ('ppo', 'classic:CartPole-v1', 'discrete', 4, 2), ('ppo', 'classic:Pendulum-v1', 'continuous', 3, 1),
    ('ddpg', 'classic:Pendulum-v1', 'continuous', 3, 1), ('dqn', 'classic:CartPole-v1', 'discrete', 4, 2)])
def test_launchers_route_classic_env_names(tmp_path, launcher, name, kind, D, A):
    from surreal_b200.main.ppo_configs import PPOLauncher
    from surreal_b200.main.ddpg_configs import DDPGLauncher
    from surreal_b200.main.dqn_configs import DQNLauncher
    la = {'ppo': PPOLauncher, 'ddpg': DDPGLauncher, 'dqn': DQNLauncher}[launcher]()
    la.setup(['--env', name, '--num-agents', '8', '--experiment-folder', str(tmp_path)])
    ec = la.env_config
    assert ec.env_name == name and ec.num_envs == 8
    assert tuple(ec.obs_spec['low_dim']['flat_inputs']) == (D,)
    assert tuple(ec.action_spec['dim']) == (A,) and ec.action_spec['type'] == kind
    assert ec.limit_episode_length == {'classic:CartPole-v1': 500, 'classic:Pendulum-v1': 200}[name]
    # synthetic names as before
    la = {'ppo': PPOLauncher, 'ddpg': DDPGLauncher, 'dqn': DQNLauncher}[launcher]()
    la.setup(['--env', 'synthetic:12:3', '--num-agents', '8', '--experiment-folder', str(tmp_path)])
    assert la.env_config.env_name == 'synthetic' and tuple(la.env_config.obs_spec['low_dim']['flat_inputs']) == (12,)
    with pytest.raises(ValueError):
        {'ppo': PPOLauncher, 'ddpg': DDPGLauncher, 'dqn': DQNLauncher}[launcher]().setup(
            ['--env', 'classic:MountainCar-v0', '--num-agents', '8', '--experiment-folder', str(tmp_path)])


def _record_args(self, num_envs, limit_episode_length=0, seed=0, device=None):
    """Constructor of the stand-ins for the device env classes (no GPU here): records its arguments."""
    self.args = (num_envs, limit_episode_length, seed)


@pytest.mark.parametrize('agent', ['base', 'ppo', 'ppo_categorical', 'q'])
def test_agents_route_classic_env_names(monkeypatch, agent):
    from surreal_b200.env import classic
    from surreal_b200.agent.base import Agent
    from surreal_b200.agent.ppo_agent import PPOAgent
    from surreal_b200.agent.q_agent import QAgent
    from surreal_b200.main.ppo_configs import PPO_DEFAULT_ENV_CONFIG, make_classic_env_config
    fakes = {k: type(v.__name__, (v,), {'__init__': _record_args}) for k, v in classic.CLASSIC_ENVS.items()}
    for k, v in fakes.items():
        monkeypatch.setitem(classic.CLASSIC_ENVS, k, v)
    name = 'classic:Pendulum-v1' if agent in ('base', 'ppo') else 'classic:CartPole-v1'
    ec = make_classic_env_config(_fresh(PPO_DEFAULT_ENV_CONFIG), name, 6, seed=9)
    ec.limit_episode_length = 37
    # an agent without its networks (they need a GPU): get_env reads only the configs and the policy type
    me = object.__new__({'base': Agent, 'ppo': PPOAgent, 'ppo_categorical': PPOAgent, 'q': QAgent}[agent])
    me.env_config, me.num_envs, me.categorical, me.action_dim, me.n_actions = ec, 6, agent != 'ppo', 2, 2
    get_env = me.get_env
    env = get_env()
    assert type(env) is fakes[name.split(':')[1]] and env.args == (6, 37, 9)
    ec.env_name = 'classic:Acrobot-v1'
    with pytest.raises(ValueError):
        get_env()
    ec.env_name = 'gym:CartPole-v1'
    with pytest.raises(ValueError):
        get_env()


def test_kernels_cross_compile_for_sm_90a(tmp_path):
    from surreal_b200 import build
    assert 'arch=compute_90a,code=sm_90a' in build.FLAGS
    if not os.path.exists(build.NVCC):
        pytest.skip('nvcc not installed')
    src = os.path.join(build.CSRC, 'env.cu')
    r = subprocess.run([build.NVCC] + build.FLAGS + ['-c', src, '-o', str(tmp_path / 'env.o')],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    # one kernel per task and variant, none spilling
    kernels = [b for b in (r.stdout + r.stderr).split('Compiling entry function')[1:] if 'classic_' in b.split('\n')[0]]
    assert len(kernels) == 6
    for b in kernels:
        assert '0 bytes spill stores, 0 bytes spill loads' in b, b
    r = subprocess.run([sys.executable, '-m', 'surreal_b200.build'], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr

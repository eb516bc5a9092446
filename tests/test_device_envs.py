"""The device envs' one routing and one descriptor: env.make_env picks the synthetic env's form from the specs for every
agent type (CPU, with stand-in env classes), and each env's sb200_env carries the key its kernels draw with and the
buffers it owns, which the persistent rollout reads through the same descriptor (GPU)."""
import copy
import ctypes as C

import pytest

from helpers import ppo_configs


def _fresh(tree):
    from surreal_b200.session import Config
    return Config(copy.deepcopy(tree.to_dict()))


def _record_args(self, num_envs, shape, action_dim, limit_episode_length, seed=0, device=None):
    """Constructor of the stand-ins for the synthetic env classes (no GPU here): records its arguments."""
    self.args = (num_envs, shape, action_dim, limit_episode_length, seed)


@pytest.mark.parametrize('agent,spec', [
    ('base', 'plain'), ('base', 'pixel'), ('ppo', 'plain'), ('ppo', 'pixel'),
    ('ppo_categorical', 'discrete'), ('ppo_categorical', 'pixel_discrete'), ('q', 'discrete')])
def test_agents_route_synthetic_env_configs(monkeypatch, agent, spec):
    import surreal_b200.env as E
    from surreal_b200.agent.base import Agent
    from surreal_b200.agent.ppo_agent import PPOAgent
    from surreal_b200.agent.q_agent import QAgent
    from surreal_b200.main.ppo_configs import (PPO_DEFAULT_ENV_CONFIG, make_synthetic_env_config,
                                               make_synthetic_pixel_env_config)
    from surreal_b200.main.dqn_configs import make_discrete_synthetic_env_config
    fakes = {k: type(k, (getattr(E, k),), {'__init__': _record_args})
             for k in ('SyntheticEnv', 'DiscreteSyntheticEnv', 'SyntheticPixelEnv')}
    for k, v in fakes.items():
        monkeypatch.setattr(E, k, v)
    ec = _fresh(PPO_DEFAULT_ENV_CONFIG)
    if spec == 'plain':
        make_synthetic_env_config(ec, 6, 12, 3, seed=9)
        want = ('SyntheticEnv', (6, 12, 3, 37, 9))
    elif spec == 'discrete':
        make_discrete_synthetic_env_config(ec, 6, 12, 5, seed=9)
        want = ('DiscreteSyntheticEnv', (6, 12, 5, 37, 9))
    else:
        make_synthetic_pixel_env_config(ec, 6, (2, 16, 16), 3, seed=9)
        if spec == 'pixel_discrete':
            ec.action_spec = {'dim': (4,), 'type': 'discrete'}
        want = ('SyntheticPixelEnv', (6, (2, 16, 16), 4 if spec == 'pixel_discrete' else 3, 37, 9))
    ec.limit_episode_length = 37
    # an agent without its networks (they need a GPU): get_env reads only the configs
    me = object.__new__({'base': Agent, 'ppo': PPOAgent, 'ppo_categorical': PPOAgent, 'q': QAgent}[agent])
    me.env_config, me.num_envs = ec, 6
    env = me.get_env()
    assert type(env) is fakes[want[0]] and env.args == want[1]
    ec.env_name = 'gym:HalfCheetah-v2'
    with pytest.raises(ValueError):
        me.get_env()


def _envs():
    from surreal_b200 import _lib
    from surreal_b200.env import CartPoleEnv, DiscreteSyntheticEnv, PendulumEnv, SyntheticEnv, SyntheticPixelEnv
    return [(SyntheticEnv(9, 12, 3, limit_episode_length=7, seed=5), _lib.ENV_SYNTH, 12),
            (DiscreteSyntheticEnv(9, 12, 4, limit_episode_length=7, seed=5), _lib.ENV_SYNTH, 12),
            (SyntheticPixelEnv(9, (2, 8, 8), 3, limit_episode_length=7, seed=5), _lib.ENV_SYNTH_PIXEL, 12),
            (CartPoleEnv(9, limit_episode_length=7, seed=5), _lib.ENV_CARTPOLE, 5),
            (PendulumEnv(9, seed=5), _lib.ENV_PENDULUM, 5)]


@pytest.mark.gpu
def test_descriptor_carries_the_kernels_key_and_the_env_buffers():
    """seed + 7 for the synthetic envs (the key the float64 rollout oracles draw with), the seed itself for the classic
    tasks; every buffer pointer is the env's own tensor, and what the kind does not use is NULL."""
    from surreal_b200 import _lib
    for env, kind, key in _envs():
        d = env.desc
        assert (d.kind, d.N, d.D, d.A, d.max_steps, d.seed) == (kind, env.N, env.D, env.A, env.max_steps, key)
        for k in ('state', 'ep_step', 'step_counter', 'obs_next', 'reward', 'done'):
            assert getattr(d, k) == getattr(env, k).data_ptr(), k
        classic = hasattr(env, 'episode')
        assert d.obs == (env.obs.data_ptr() if classic else None)
        assert d.episode == (env.episode.data_ptr() if classic else None)
        synth = kind == _lib.ENV_SYNTH
        assert (d.WsT, d.WaT) == ((env.WsT.data_ptr(), env.WaT.data_ptr()) if synth else (None, None))


@pytest.mark.gpu
def test_rollout_args_point_at_the_envs_own_descriptor():
    from surreal_b200.agent import PPOAgent
    from surreal_b200.env import SyntheticEnv
    from surreal_b200.replay import FIFOReplay
    N, D, A = 32, 8, 2
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=(32, 32), n_step=4, stride=4, B=N)   # a policy the kernel takes
    ec.num_envs = N
    FIFOReplay(lc, ec, sc)
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    env = SyntheticEnv(N, D, A, limit_episode_length=9, seed=3)
    ag.env = w = ag.prepare_env_agent(env)
    assert ag.rollout_chunk_supported()
    for a in (ag._rollout_args(), ag._rollout_args(w.rollout_outbox(8), 8)):
        assert C.addressof(a.env.contents) == C.addressof(env.desc)


@pytest.mark.gpu
def test_step_takes_only_the_action_rows_of_its_actors():
    """Every env checks the tensor it passes to its kernel: float32, contiguous, on the device, [N, A] rows -- or [A]
    for a single actor, as the agents return it."""
    import torch
    from surreal_b200.env import SyntheticEnv
    for env, _, _ in _envs():
        env.reset()
        a = torch.zeros(env.N, env.A, device='cuda')
        env.step(a)
        env.step((a, None))                                      # QAgent.act's (one-hot rows, indices)
        strided = torch.zeros(env.N, env.A + 1, device='cuda')[:, :env.A]
        for bad in (a.double(), a.cpu(), strided, a[:-1], a.view(-1)):
            with pytest.raises(ValueError):
                env.step(bad)
    one = SyntheticEnv(1, 12, 3, seed=5)
    one.reset()
    one.step(torch.zeros(3, device='cuda'))
    with pytest.raises(ValueError):
        one.step(torch.zeros(2, device='cuda'))

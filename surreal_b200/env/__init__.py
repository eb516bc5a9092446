from .base import DeviceEnv  # noqa: F401
from .synthetic import SyntheticEnv, SyntheticPixelEnv, DiscreteSyntheticEnv  # noqa: F401
from .classic import CartPoleEnv, PendulumEnv, make_classic_env  # noqa: F401
from .exp_sender_wrapper import (ExpSenderWrapperMultiStepMovingWindowWithInfo,  # noqa: F401
                                 ExpSenderWrapperSSARNStepBootstrap)


def make_env(env_config, num_envs):
    """The in-tree device env of ``env_config`` for ``num_envs`` actors: a ``classic:<task>`` name gives that task; any
    other name must start with ``synthetic``, and the specs pick the synthetic env's form -- pixel frames for a pixel
    obs_spec, one-hot action rows for a discrete action_spec, else continuous actions."""
    from ..utils import action_is_discrete, obs_is_pixel
    ec = env_config
    env = make_classic_env(ec, num_envs)
    if env is not None:
        return env
    name = ec.env_name if 'env_name' in ec else ''
    if not str(name).startswith('synthetic'):
        raise ValueError('only the device-resident envs ship with surreal_b200 (env_name "synthetic", '
                         '"classic:CartPole-v1", "classic:Pendulum-v1"); '
                         'gym / dm_control / robosuite adapters are out of scope -- pass your own env to '
                         'main_setup(env)')
    seed = int(ec.seed) if 'seed' in ec else 0
    A = ec.action_spec.dim[0]
    if obs_is_pixel(ec.obs_spec):
        return SyntheticPixelEnv(num_envs, tuple(ec.obs_spec['pixel']['camera0']), A, ec.limit_episode_length, seed=seed)
    D = sum(v[0] for v in ec.obs_spec['low_dim'].values())
    if action_is_discrete(ec.action_spec):
        return DiscreteSyntheticEnv(num_envs, D, A, ec.limit_episode_length, seed=seed)
    return SyntheticEnv(num_envs, D, A, ec.limit_episode_length, seed=seed)

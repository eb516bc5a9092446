"""PPO default config trees + launcher wiring (behavioural mirror of surreal/main/ppo_configs.py:15-228).
Hyper-parameter values are the contract with existing experiments; equality with the reference's
trees is pinned by tests/test_default_configs.py."""
import argparse

from ..session import Config, LOCAL_SESSION_CONFIG, BASE_LEARNER_CONFIG, BASE_ENV_CONFIG

PPO_DEFAULT_LEARNER_CONFIG = Config({
    'model': {'convs': [], 'actor_fc_hidden_sizes': [300, 200], 'critic_fc_hidden_sizes': [300, 200],
              'cnn_feature_dim': 256, 'use_layernorm': False},
    'algo': {
        'use_z_filter': True, 'use_r_filter': False, 'gamma': .995, 'n_step': 25, 'stride': 20,
        'network': {
            'lr_actor': 1e-4, 'lr_critic': 1e-4,
            'clip_actor_gradient': True, 'actor_gradient_norm_clip': 5.,
            'clip_critic_gradient': True, 'critic_gradient_norm_clip': 5.,
            'actor_regularization': 0.0, 'critic_regularization': 0.0,
            'anneal': {'lr_scheduler': 'LinearWithMinLR', 'frames_to_anneal': 5e6, 'lr_update_frequency': 100,
                       'min_lr': 5e-5},
        },
        'ppo_mode': 'adapt',
        'advantage': {'norm_adv': True, 'lam': 0.97, 'reward_scale': 1.0},
        'rnn': {'if_rnn_policy': True, 'rnn_hidden': 100, 'rnn_layer': 1, 'horizon': 5},
        'consts': {'init_log_sig': -1.0, 'log_sig_range': 0.25, 'epoch_policy': 10, 'epoch_baseline': 10,
                   'adjust_threshold': (0.5, 2.0), 'kl_target': 0.015},
        'adapt_consts': {'kl_cutoff_coeff': 250, 'beta_init': 1.0, 'beta_range': (1 / 35.0, 35.0),
                         'scale_constant': 1.5},
        'clip_consts': {'clip_epsilon_init': 0.2, 'clip_range': (0.05, 0.3), 'scale_constant': 1.2},
    },
    'replay': {'batch_size': 64, 'memory_size': 96, 'sampling_start_size': 64, 'replay_shards': 1},
    'parameter_publish': {'exp_interval': 4096},
})
PPO_DEFAULT_LEARNER_CONFIG.extend(BASE_LEARNER_CONFIG)

PPO_DEFAULT_ENV_CONFIG = Config({
    'env_name': '', 'action_repeat': 1, 'pixel_input': False, 'use_grayscale': False, 'use_depth': False,
    'frame_stacks': 1, 'sleep_time': 0,
    'video': {'record_video': False, 'save_folder': None, 'max_videos': 500, 'record_every': 5},
    'observation': {'pixel': ['camera0'], 'low_dim': ['robot-state', 'object-state']},
    'eval_mode': {'demonstration': None},
    'demonstration': {
        'use_demo': False, 'adaptive': True, 'increment_frequency': 100, 'sample_window_width': 25, 'increment': 25,
        'mixing': ['random'], 'mixing_ratio': [1.0], 'ratio_step': [0.0], 'improve_threshold': 0.1,
        'curriculum_length': 50, 'history_length': 20,
    },
    'limit_episode_length': 200, 'stochastic_eval': True,
})
PPO_DEFAULT_ENV_CONFIG.extend(BASE_ENV_CONFIG)

PPO_DEFAULT_SESSION_CONFIG = Config({
    'folder': '_str_',
    'tensorplex': {'update_schedule': {'training_env': 20, 'eval_env': 5, 'eval_env_sleep': 2, 'agent': 50,
                                       'learner': 20}},
    'agent': {'fetch_parameter_mode': 'step', 'fetch_parameter_interval': 100, 'num_gpus': 0},
    'sender': {'flush_iteration': 3},
    'learner': {'num_gpus': 0},
    'replay': {'max_puller_queue': 3, 'max_prefetch_queue': 1},
    'checkpoint': {'learner': {'mode': 'history', 'periodic': 1000, 'min_interval': 15 * 60}},
})
PPO_DEFAULT_SESSION_CONFIG.extend(LOCAL_SESSION_CONFIG)


def ppo_argparser():
    """The `-- <flags>` accepted after the component name (ppo_configs.py:194-209)."""
    p = argparse.ArgumentParser()
    p.add_argument('--env', type=str, required=True)
    p.add_argument('--num-agents', type=int, required=True)
    p.add_argument('--num-gpus', type=int, default=0)
    p.add_argument('--agent-num-gpus', type=int, default=0)
    p.add_argument('--restore-folder', type=str, default=None)
    p.add_argument('--experiment-folder', required=True)
    p.add_argument('--agent-batch', type=int, default=1)
    p.add_argument('--unit-test', action='store_true')
    return p


def make_synthetic_env_config(env_config, num_envs, obs_dim=64, action_dim=8, seed=0):
    """What surreal.env.make_env_config does for a real env (ppo_configs.py:213-214): fill obs_spec /
    action_spec.  Here for the device-resident synthetic env of the benchmark configs."""
    env_config.env_name = 'synthetic'
    env_config.num_envs = int(num_envs)
    env_config.seed = int(seed)
    env_config.obs_spec = {'low_dim': {'flat_inputs': (obs_dim,)}}
    env_config.action_spec = {'dim': (action_dim,), 'type': 'continuous'}
    return env_config


def make_classic_env_config(env_config, name, num_envs, seed=0):
    """obs_spec / action_spec of a classic-control task (``name`` = 'classic:CartPole-v1' or 'classic:Pendulum-v1',
    env.classic), and limit_episode_length = the task's registered limit (500 / 200), which the PPO env tree's 200 would
    otherwise cut short; a caller may override it afterwards."""
    from ..env.classic import classic_env_class
    cls = classic_env_class(name)
    if cls is None:
        raise ValueError('%r is not a classic-control env name (classic:<task>)' % (name,))
    env_config.env_name = str(name)
    env_config.num_envs = int(num_envs)
    env_config.seed = int(seed)
    env_config.obs_spec = {'low_dim': {'flat_inputs': (cls.D,)}}
    env_config.action_spec = {'dim': (cls.A,), 'type': cls.ACTION_TYPE}
    env_config.limit_episode_length = cls.MAX_STEPS
    return env_config


def make_synthetic_pixel_env_config(env_config, num_envs, frame_shape=(4, 84, 84), action_dim=8, seed=0):
    """Pixel flavour (BASELINE configs[3]): obs_spec = {'pixel': {'camera0': (C, H, W)}}, pixel_input on -- what
    surreal.env.make_env_config fills in for a pixel env (docs/env.md:79-108)."""
    env_config.env_name = 'synthetic-pixel'
    env_config.num_envs = int(num_envs)
    env_config.seed = int(seed)
    env_config.pixel_input = True
    env_config.obs_spec = {'pixel': {'camera0': tuple(int(v) for v in frame_shape)}}
    env_config.action_spec = {'dim': (action_dim,), 'type': 'continuous'}
    return env_config


class PPOLauncher:
    """PPOLauncher of ppo_configs.py:178-228 (constructed lazily so importing configs needs no GPU)."""

    def __new__(cls, *a, **k):
        from ..launch import SurrealDefaultLauncher
        from ..agent import PPOAgent
        from ..learner import PPOLearner
        from ..replay import FIFOReplay

        class _PPOLauncher(SurrealDefaultLauncher):
            def __init__(self):
                super().__init__(PPOAgent, PPOLearner, FIFOReplay, PPO_DEFAULT_SESSION_CONFIG.copy(),
                                 PPO_DEFAULT_ENV_CONFIG.copy(), PPO_DEFAULT_LEARNER_CONFIG.copy())

            def setup(self, argv):
                args = ppo_argparser().parse_args(args=argv)
                name = args.env
                if name.startswith('classic:'):
                    make_classic_env_config(self.env_config, name, args.num_agents)
                else:
                    dims = name.split(':')[1:] if ':' in name else []
                    D = int(dims[0]) if len(dims) > 0 else 64
                    A = int(dims[1]) if len(dims) > 1 else 8
                    make_synthetic_env_config(self.env_config, args.num_agents, D, A)
                self.session_config.folder = args.experiment_folder
                self.session_config.agent.num_gpus = args.agent_num_gpus
                self.session_config.learner.num_gpus = args.num_gpus
                if args.restore_folder is not None:
                    self.session_config.checkpoint.restore = True
                    self.session_config.checkpoint.restore_folder = args.restore_folder
                self.agent_batch_size = args.agent_batch
                self.eval_batch_size = args.agent_batch
                if args.unit_test:
                    self.learner_config.replay.batch_size = 2
                    self.learner_config.replay.sampling_start_size = 2
        return _PPOLauncher()


def main():
    PPOLauncher().main()

"""DDPG default config trees (behavioural mirror of surreal/main/ddpg_configs.py:16-174); pinned against the
reference's trees by tests/test_default_configs.py."""
import argparse

from ..session import Config, LOCAL_SESSION_CONFIG, BASE_LEARNER_CONFIG, BASE_ENV_CONFIG

DDPG_DEFAULT_LEARNER_CONFIG = Config({
    'model': {
        'convs': [], 'actor_fc_hidden_sizes': [300, 200], 'critic_fc_hidden_sizes': [400, 300],
        'use_layernorm': False,
        'conv_spec': {'out_channels': [16, 32], 'kernel_sizes': [8, 4], 'strides': [4, 2],
                      'hidden_output_dim': 200},
    },
    'algo': {
        'gamma': .99, 'n_step': 3, 'stride': 1,
        'network': {
            'lr_actor': 1e-4, 'lr_critic': 1e-3,
            'clip_actor_gradient': True, 'actor_gradient_value_clip': 1.,
            'clip_critic_gradient': False, 'critic_gradient_value_clip': 5.,
            'actor_regularization': 0.0, 'critic_regularization': 0.0,
            'use_action_regularization': False, 'use_double_critic': False,
            'target_update': {'type': 'hard', 'interval': 500},
        },
        'exploration': {
            'param_noise_type': None, 'param_noise_sigma': 0.05, 'param_noise_alpha': 1.15,
            'param_noise_target_stddev': 0.005, 'noise_type': 'normal', 'max_sigma': 1.0, 'theta': 0.15,
            'dt': 1e-3,
        },
    },
    'replay': {'batch_size': 512, 'memory_size': int(1000000 / 3), 'sampling_start_size': 3000, 'replay_shards': 3},
    'parameter_publish': {'min_publish_interval': 3},
})
DDPG_DEFAULT_LEARNER_CONFIG.extend(BASE_LEARNER_CONFIG)

DDPG_DEFAULT_ENV_CONFIG = Config({
    'env_name': '_str_', 'num_agents': '_int_', 'demonstration': None, 'use_depth': False, 'render': False,
    'use_demonstration': False, 'pixel_input': False, 'use_grayscale': False, 'frame_stacks': 3,
    'action_repeat': 1, 'frame_stack_concatenate_on_env': False, 'sleep_time': 0.0, 'limit_episode_length': 0,
    'video': {'record_video': True, 'save_folder': None, 'max_videos': 500, 'record_every': 20},
    'observation': {
        'pixel': ['camera0', 'depth'],
        'low_dim': ['position', 'velocity', 'proprio', 'robot-state', 'cube_pos', 'cube_quat', 'gripper_to_cube',
                    'low-dim'],
    },
})
DDPG_DEFAULT_ENV_CONFIG.extend(BASE_ENV_CONFIG)

DDPG_DEFAULT_SESSION_CONFIG = Config({
    'folder': '_str_',
    'tensorplex': {'update_schedule': {'training_env': 20, 'eval_env': 5, 'eval_env_sleep': 30, 'agent': 50,
                                       'learner': 20}},
    'agent': {'fetch_parameter_mode': 'step', 'fetch_parameter_interval': 200, 'num_gpus': 0},
    'sender': {'flush_iteration': 100},
    'learner': {'prefetch_processes': 3, 'num_gpus': 0},
})
DDPG_DEFAULT_SESSION_CONFIG.extend(LOCAL_SESSION_CONFIG)


def ddpg_argparser():
    """ddpg_configs.py:249-271."""
    p = argparse.ArgumentParser()
    p.add_argument('--env', type=str, required=True)
    p.add_argument('--num-agents', type=int, required=True)
    p.add_argument('--num-gpus', type=int, default=0)
    p.add_argument('--agent-num-gpus', type=int, default=0)
    p.add_argument('--restore-folder', type=str, default=None)
    p.add_argument('--experiment-folder', required=True)
    p.add_argument('--agent-batch', type=int, default=1)
    p.add_argument('--eval-batch', type=int, default=1)
    p.add_argument('--unit-test', action='store_true')
    # the single-GPU engine (launch.ReplayEngine): env steps per actor chunk, learner updates beside each chunk (default:
    # one per env step), and an optional cap on engine steps (default: run until interrupted)
    p.add_argument('--rollout-steps', type=int, default=None)
    p.add_argument('--updates-per-chunk', type=int, default=None)
    p.add_argument('--iterations', type=int, default=None)
    # proportional prioritized replay (replay.PrioritizedReplay) instead of the uniform ring; its alpha, beta0,
    # beta_anneal_iters and priority_eps come from learner_config.replay when set there
    p.add_argument('--prioritized-replay', action='store_true')
    return p


class DDPGLauncher:
    """DDPGLauncher of ddpg_configs.py:230-293 (constructed lazily so importing configs needs no GPU)."""

    def __new__(cls, *a, **k):
        from ..launch import SurrealDefaultLauncher
        from ..agent import DDPGAgent
        from ..learner import DDPGLearner
        from ..replay import UniformReplay, PrioritizedReplay
        from .ppo_configs import make_synthetic_env_config, make_classic_env_config

        class _DDPGLauncher(SurrealDefaultLauncher):
            def __init__(self):
                super().__init__(DDPGAgent, DDPGLearner, UniformReplay, DDPG_DEFAULT_SESSION_CONFIG.copy(),
                                 DDPG_DEFAULT_ENV_CONFIG.copy(), DDPG_DEFAULT_LEARNER_CONFIG.copy())

            def setup(self, argv):
                args = ddpg_argparser().parse_args(args=argv)
                if args.env.startswith('classic:'):
                    make_classic_env_config(self.env_config, args.env, args.num_agents)
                else:
                    dims = args.env.split(':')[1:] if ':' in args.env else []
                    D = int(dims[0]) if len(dims) > 0 else 64
                    A = int(dims[1]) if len(dims) > 1 else 8
                    make_synthetic_env_config(self.env_config, args.num_agents, D, A)
                self.env_config.num_agents = args.num_agents
                self.session_config.folder = args.experiment_folder
                self.session_config.agent.num_gpus = args.agent_num_gpus
                self.session_config.learner.num_gpus = args.num_gpus
                if args.restore_folder is not None:
                    self.session_config.checkpoint.restore = True
                    self.session_config.checkpoint.restore_folder = args.restore_folder
                self.agent_batch_size = args.agent_batch
                self.eval_batch_size = args.eval_batch
                self.rollout_steps, self.updates_per_chunk = args.rollout_steps, args.updates_per_chunk
                self.iterations = args.iterations
                if args.prioritized_replay:
                    self.replay_class = PrioritizedReplay
                if args.unit_test:
                    self.learner_config.replay.sampling_start_size = 5
                    self.learner_config.replay.replay_shards = 1
                    self.session_config.ps.shards = 1
        return _DDPGLauncher()


def main():
    DDPGLauncher().main()

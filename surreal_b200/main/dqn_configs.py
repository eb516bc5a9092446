"""DQN default config trees: DQNLearner.default_config (surreal/learner/dqn.py:94-121) merged with QAgent.default_config
(surreal/agent/q_agent.py:55-65).  The reference's required placeholders (model.fc_hidden_sizes / dueling / convs,
algo.target_network_update_freq, algo.exploration.steps, eval.eps) stay required: a run fills them in."""
import argparse

from ..session import Config, BASE_LEARNER_CONFIG
from .ddpg_configs import DDPG_DEFAULT_ENV_CONFIG, DDPG_DEFAULT_SESSION_CONFIG
from .ppo_configs import make_classic_env_config

DQN_DEFAULT_LEARNER_CONFIG = Config({
    'model': {'convs': '_list_', 'fc_hidden_sizes': '_list_', 'dueling': '_bool_'},
    'algo': {
        'lr': 1e-3, 'optimizer': 'Adam', 'grad_norm_clipping': 10, 'gamma': .99,
        'target_network_update_freq': '_int_', 'double_q': True,
        'exploration': {'schedule': 'linear', 'steps': '_int_', 'final_eps': 0.01},
        'prioritized': {'enabled': False, 'alpha': 0.6, 'beta0': 0.4, 'beta_anneal_iters': None, 'eps': 1e-6},
    },
    'eval': {'eps': '_float_'},
    # not in the reference's DQN tree (its replay config came from the session); values as DDPG's tree has them
    'replay': {'batch_size': 512, 'memory_size': 1000000, 'sampling_start_size': 10000},
    'parameter_publish': {'min_publish_interval': 3},
})
DQN_DEFAULT_LEARNER_CONFIG.extend(BASE_LEARNER_CONFIG)

DQN_DEFAULT_ENV_CONFIG = DDPG_DEFAULT_ENV_CONFIG.copy()
DQN_DEFAULT_SESSION_CONFIG = DDPG_DEFAULT_SESSION_CONFIG.copy()


def make_discrete_synthetic_env_config(env_config, num_envs, obs_dim=64, n_actions=18, seed=0):
    """obs_spec / action_spec of the device-resident discrete synthetic env (env.DiscreteSyntheticEnv)."""
    env_config.env_name = 'synthetic'
    env_config.num_envs = int(num_envs)
    env_config.seed = int(seed)
    env_config.obs_spec = {'low_dim': {'flat_inputs': (obs_dim,)}}
    env_config.action_spec = {'dim': (n_actions,), 'type': 'discrete'}
    return env_config


def dqn_argparser():
    p = argparse.ArgumentParser()
    p.add_argument('--env', type=str, required=True)            # synthetic[:D[:n_actions]] or classic:CartPole-v1
    p.add_argument('--num-agents', type=int, required=True)
    p.add_argument('--experiment-folder', required=True)
    p.add_argument('--restore-folder', type=str, default=None)
    p.add_argument('--fc-hidden-sizes', type=int, nargs='+', default=[256, 256])
    p.add_argument('--no-dueling', action='store_true')
    p.add_argument('--target-update-freq', type=int, default=10000)      # samples
    p.add_argument('--exploration-steps', type=int, default=100000)
    p.add_argument('--eval-eps', type=float, default=0.05)
    p.add_argument('--batch-size', type=int, default=None)
    p.add_argument('--memory-size', type=int, default=None)
    p.add_argument('--sampling-start-size', type=int, default=None)
    # the single-GPU engine (launch.ReplayEngine) and proportional prioritized replay (algo.prioritized.enabled)
    p.add_argument('--rollout-steps', type=int, default=None)
    p.add_argument('--updates-per-chunk', type=int, default=None)
    p.add_argument('--iterations', type=int, default=None)
    p.add_argument('--prioritized-replay', action='store_true')
    return p


class DQNLauncher:
    """Launcher for QAgent + DQNLearner on the device-resident discrete synthetic env (constructed lazily so importing
    configs needs no GPU).  algo.prioritized.enabled selects PrioritizedReplay, else UniformReplay."""

    def __new__(cls, *a, **k):
        from ..launch import SurrealDefaultLauncher
        from ..agent import QAgent
        from ..learner import DQNLearner
        from ..replay import UniformReplay, PrioritizedReplay

        class _DQNLauncher(SurrealDefaultLauncher):
            def __init__(self):
                super().__init__(QAgent, DQNLearner, UniformReplay, DQN_DEFAULT_SESSION_CONFIG.copy(),
                                 DQN_DEFAULT_ENV_CONFIG.copy(), DQN_DEFAULT_LEARNER_CONFIG.copy())

            def setup(self, argv):
                args = dqn_argparser().parse_args(args=argv)
                if args.env.startswith('classic:'):
                    make_classic_env_config(self.env_config, args.env, args.num_agents)
                else:
                    dims = args.env.split(':')[1:] if ':' in args.env else []
                    D = int(dims[0]) if len(dims) > 0 else 64
                    n = int(dims[1]) if len(dims) > 1 else 18
                    make_discrete_synthetic_env_config(self.env_config, args.num_agents, D, n)
                self.env_config.num_agents = args.num_agents
                lc = self.learner_config
                lc.model.convs, lc.model.fc_hidden_sizes = [], list(args.fc_hidden_sizes)
                lc.model.dueling = not args.no_dueling
                lc.algo.target_network_update_freq = args.target_update_freq
                lc.algo.exploration.steps = args.exploration_steps
                lc.eval.eps = args.eval_eps
                for k in ('batch_size', 'memory_size', 'sampling_start_size'):
                    if getattr(args, k) is not None:
                        lc.replay[k] = getattr(args, k)
                lc.algo.prioritized.enabled = bool(args.prioritized_replay)
                if lc.algo.prioritized.enabled:
                    self.replay_class = PrioritizedReplay
                self.session_config.folder = args.experiment_folder
                if args.restore_folder is not None:
                    self.session_config.checkpoint.restore = True
                    self.session_config.checkpoint.restore_folder = args.restore_folder
                self.rollout_steps, self.updates_per_chunk = args.rollout_steps, args.updates_per_chunk
                self.iterations = args.iterations
        return _DQNLauncher()


def main():
    DQNLauncher().main()

"""TEST INFRASTRUCTURE -- the learning runs of the classic-control tasks: one committed config per algorithm family, a
training loop through the library's own engines, and the evaluation the learning tests and
tools/classic_control_train.py share.

Evaluation: a fresh env with another seed, an agent in eval_deterministic mode that loads the learner's weights as a
parameter fetch would (without a publish, so evaluating does not change the run), and the return of every actor's FIRST episode, summed here from the env's reward and done
tensors.  Nothing in the library monitors episodes.

Each case lists where its config departs from the reference defaults (surreal/main/*_configs.py, mirrored by
surreal_b200/main/*_configs.py)."""
import copy
import tempfile
import time

import numpy as np
import torch

EVAL_SEED = 1234567
EVAL_ACTORS = 64


def _trees(kind):
    from surreal_b200.session import Config
    if kind == 'ppo':
        from surreal_b200.main.ppo_configs import (PPO_DEFAULT_LEARNER_CONFIG as L, PPO_DEFAULT_ENV_CONFIG as E,
                                                   PPO_DEFAULT_SESSION_CONFIG as S)
    elif kind == 'ddpg':
        from surreal_b200.main.ddpg_configs import (DDPG_DEFAULT_LEARNER_CONFIG as L, DDPG_DEFAULT_ENV_CONFIG as E,
                                                    DDPG_DEFAULT_SESSION_CONFIG as S)
    else:
        from surreal_b200.main.dqn_configs import (DQN_DEFAULT_LEARNER_CONFIG as L, DQN_DEFAULT_ENV_CONFIG as E,
                                                   DQN_DEFAULT_SESSION_CONFIG as S)
    lc, ec, sc = (Config(copy.deepcopy(t.to_dict())) for t in (L, E, S))
    sc.folder = tempfile.mkdtemp()
    return lc, ec, sc


def _env(ec, name, N, seed):
    from surreal_b200.main.ppo_configs import make_classic_env_config
    make_classic_env_config(ec, name, N, seed)
    ec.num_agents = N


class Case:
    """One learning run: ``kind`` ppo / ddpg / dqn, the env name, the configs, and the engine shape."""

    def __init__(self, name, kind, env, build, T, K=None, bar=None, random_below=None):
        self.name, self.kind, self.env, self.build, self.T, self.K = name, kind, env, build, T, K
        self.bar, self.random_below = bar, random_below

    def configs(self, seed=0):
        lc, ec, sc = _trees(self.kind)
        self.build(lc, ec, sc, seed)
        return lc, ec, sc


# -- the committed configs ---------------------------------------------------------------------------------------------
def _ppo_cartpole_mlp(lc, ec, sc, seed):
    """Categorical PPO, MLP policy: the default PPO config (adapt mode, batch 64, lr 1e-4, 300-200 layers) with the LSTM
    off, windows of 8 steps with stride 4 instead of 25 / 20 (a window never spans two episodes, and an untrained
    policy's episodes last about 10 to 20 steps), and no wall-clock publish throttle; 64 actors."""
    _env(ec, 'classic:CartPole-v1', 64, seed)
    lc.algo.rnn.if_rnn_policy = False
    lc.algo.n_step, lc.algo.stride = 8, 4
    lc.replay.memory_size = 4096
    lc.parameter_publish.min_publish_interval = 0.0


def _ppo_cartpole_default(lc, ec, sc, seed):
    """The default PPO config (adapt mode, LSTM policy, n_step 25, stride 20, batch 64, lr 1e-4) with one change: no
    wall-clock publish throttle (0.3 s by default), so that the run depends on its seed alone.  The run's shape: 64
    actors (one batch per 20-step chunk) and CartPole's registered episode limit."""
    _env(ec, 'classic:CartPole-v1', 64, seed)
    lc.parameter_publish.min_publish_interval = 0.0


def _ppo_pendulum(lc, ec, sc, seed):
    """Gaussian PPO, MLP policy.  Departures: no LSTM, clip mode, two 64-wide layers, lr 3e-4, gamma 0.99 / lambda 0.95,
    windows of 40 steps with stride 40 (five per 200-step episode), 512 actors and one window per actor per batch,
    a publish after every batch, fetch every chunk, no publish throttle."""
    _env(ec, 'classic:Pendulum-v1', 512, seed)
    lc.algo.rnn.if_rnn_policy = False
    lc.algo.ppo_mode = 'clip'
    lc.model.actor_fc_hidden_sizes = lc.model.critic_fc_hidden_sizes = [64, 64]
    lc.algo.network.lr_actor = lc.algo.network.lr_critic = 3e-4
    lc.algo.gamma, lc.algo.advantage.lam = 0.99, 0.95
    lc.algo.n_step = lc.algo.stride = 40
    lc.replay.batch_size, lc.replay.memory_size = 512, 1024
    lc.parameter_publish.exp_interval = 512
    sc.agent.fetch_parameter_interval = 40
    lc.parameter_publish.min_publish_interval = 0.0


def _ddpg_pendulum(lc, ec, sc, seed):
    """DDPG.  Departures from the DDPG defaults: 16 actors, two 64-wide layers in both nets, a replay of 100 000
    records starting at 2 000 with batches of 256, fetch every chunk, no publish throttle."""
    _env(ec, 'classic:Pendulum-v1', 16, seed)
    lc.model.actor_fc_hidden_sizes = lc.model.critic_fc_hidden_sizes = [64, 64]
    lc.replay.batch_size, lc.replay.memory_size, lc.replay.sampling_start_size = 256, 100000, 2000
    sc.agent.fetch_parameter_interval = 32
    lc.parameter_publish.min_publish_interval = 0.0


def _dqn_cartpole(lc, ec, sc, seed):
    """DQN (its tree's required fields filled in): dueling double-Q, two 64-wide layers, 64 actors, a target copy
    every 20 000 samples, epsilon from 1 to 0.01 over the first 1 000 batched steps, a replay of 100 000 records
    starting at 2 000 with batches of 128, fetch every chunk, no publish throttle."""
    _env(ec, 'classic:CartPole-v1', 64, seed)
    lc.model.convs, lc.model.fc_hidden_sizes, lc.model.dueling = [], [64, 64], True
    lc.algo.target_network_update_freq = 20000
    lc.algo.exploration.steps = 1000
    lc.eval.eps = 0.0
    lc.replay.batch_size, lc.replay.memory_size, lc.replay.sampling_start_size = 128, 100000, 2000
    sc.agent.fetch_parameter_interval = 8
    lc.parameter_publish.min_publish_interval = 0.0


CASES = {
    'ppo_cartpole_mlp': Case('ppo_cartpole_mlp', 'ppo', 'classic:CartPole-v1', _ppo_cartpole_mlp, T=20,
                             bar=475.0, random_below=100.0),
    'ppo_cartpole_default': Case('ppo_cartpole_default', 'ppo', 'classic:CartPole-v1', _ppo_cartpole_default, T=20,
                                 bar=195.0, random_below=100.0),
    'dqn_cartpole': Case('dqn_cartpole', 'dqn', 'classic:CartPole-v1', _dqn_cartpole, T=8, K=8,
                         bar=195.0, random_below=100.0),
    'ddpg_pendulum': Case('ddpg_pendulum', 'ddpg', 'classic:Pendulum-v1', _ddpg_pendulum, T=32, K=32,
                          bar=-250.0, random_below=-800.0),
    'ppo_pendulum': Case('ppo_pendulum', 'ppo', 'classic:Pendulum-v1', _ppo_pendulum, T=40,
                         bar=-250.0, random_below=-800.0),
}


def _classes(kind):
    from surreal_b200 import agent, learner, replay
    return {'ppo': (agent.PPOAgent, learner.PPOLearner, replay.FIFOReplay),
            'ddpg': (agent.DDPGAgent, learner.DDPGLearner, replay.UniformReplay),
            'dqn': (agent.QAgent, learner.DQNLearner, replay.UniformReplay)}[kind]


class Run:
    """A training run of one case through the launcher's objects and the engine run_engine would pick: ReplayEngine for
    DDPG and DQN, PipelinedEngine where one chunk yields one PPO batch, else chunk / learn alternation."""

    def __init__(self, case, seed=0):
        from surreal_b200.launch import SurrealDefaultLauncher, PipelinedEngine, ReplayEngine
        self.case = case
        self.lc, self.ec, self.sc = case.configs(seed)
        torch.manual_seed(seed)
        np.random.seed(seed)
        Agent, Learner, Replay = _classes(case.kind)
        self.la = SurrealDefaultLauncher(Agent, Learner, Replay, self.sc, self.ec, self.lc)
        self.la.setup_replay(0)
        self.la.setup_learner()
        np.random.seed(seed)             # the per-actor exploration constants (setup_agent would seed from the clock)
        self.la.agent = Agent(learner_config=self.lc, env_config=self.ec, session_config=self.sc, agent_id=0,
                              agent_mode='training')
        self.agent, self.replay, self.learner = self.la.setup_engine()
        self.env_steps = 0
        self.eng = None
        lc, N, T = self.lc, self.agent.num_envs, case.T
        if case.kind in ('ddpg', 'dqn'):
            self.eng = ReplayEngine(self.agent, self.replay, self.learner, T, case.K)
        elif lc.algo.n_step == lc.algo.stride == T and lc.replay.batch_size == N:
            self.eng = PipelinedEngine(self.agent, self.replay, self.learner, T)
        if self.eng is not None:
            self.eng.prime()
            self.env_steps += N * T
        self._eval = None

    def step(self):
        """One engine step (or, for the alternation, one chunk and the learner iterations it feeds)."""
        N, T = self.agent.num_envs, self.case.T
        if self.eng is not None:
            self.eng.step()
        else:
            self.agent.main_loop(max_steps=T)
            while self.replay.start_sample_condition():
                self.learner.main_loop()
        self.env_steps += N * T

    def sync(self):
        torch.cuda.synchronize()

    def evaluate(self, seed=EVAL_SEED, N=EVAL_ACTORS):
        """Mean and per-actor returns of the first episode of N fresh actors, acting with the learner's weights."""
        from surreal_b200.distributed import ModuleDict
        from surreal_b200.env import make_classic_env
        from surreal_b200.session import Config
        self.sync()
        if self._eval is None:
            Agent = _classes(self.case.kind)[0]
            ec = Config(copy.deepcopy(self.ec.to_dict()))
            ec.num_envs = ec.num_agents = N
            ec.seed = seed
            ec.stochastic_eval = False
            ag = Agent(learner_config=self.lc, env_config=ec, session_config=self.sc, agent_id=1,
                       agent_mode='eval_deterministic_local')
            self._eval = (ag, ec)
        ag, ec = self._eval
        # the learner's weights as a fetch would load them, without a publish: the run's actors see only its own
        ModuleDict(ag.module_dict()).load(ModuleDict(self.learner.module_dict()).dumps())
        if hasattr(ag, 'reset'):
            ag.reset()
        return episode_returns(ag, make_classic_env(ec, N))


def episode_returns(agent, env):
    """Each actor's first-episode return, from the env's reward and done tensors -> (mean, numpy [N])."""
    obs, _ = env.reset()
    ret = torch.zeros(env.N, dtype=torch.float64, device=env.device)
    alive = torch.ones(env.N, dtype=torch.bool, device=env.device)
    for _ in range(env.max_steps):
        obs, r, d, _ = env.step(agent.act(obs))
        ret += torch.where(alive, r.double(), torch.zeros_like(ret))
        alive &= d == 0
    assert not bool(alive.any()), 'every first episode ends by the cap'
    out = ret.cpu().numpy()
    return float(out.mean()), out


def train(case, iterations, eval_every=None, log=None, seed=0, max_seconds=None):
    """Train ``case`` for ``iterations`` engine steps.  Returns (run, curve): curve rows (env steps, training seconds,
    mean first-episode return), one before training and then every ``eval_every`` steps; training seconds exclude the
    evaluations.  ``max_seconds``: stop early once training has taken that long."""
    run = Run(case, seed)
    curve = []

    def point(spent):
        curve.append((run.env_steps, spent, run.evaluate()[0]))
        if log:
            log(case.name, *curve[-1])
    if eval_every is not None:
        point(0.0)
    spent = 0.0
    for it in range(1, iterations + 1):
        t0 = time.perf_counter()
        run.step()
        run.sync()
        spent += time.perf_counter() - t0
        last = it == iterations or (max_seconds is not None and spent >= max_seconds)
        if eval_every is not None and (it % eval_every == 0 or last):
            point(spent)
        if last:
            break
    return run, curve

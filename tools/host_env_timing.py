#!/usr/bin/env python
"""Actor loop with a batched HOST env (numpy in / numpy out), one C call per act() and per wrapper step:

    obs, _ = w.reset(); then T x (a = agent.act(obs); obs, r, d, info = w.step(a))

Rows (1024 actors, 64-dim observations, 8 actions, episodes of T = 128 steps):
  ff     feed-forward PPO at BASELINE configs[1] sizes (2x256 MLP, windows of 128), each episode followed by
         learner.main_loop() -- the same loop as bench.py's `e2e` row, so the two numbers can be compared;
  rnn1   RNN-mode PPO at the default config (LSTM(100), heads 300-200), actor loop only;
  rnn2   the same with rnn_layer = 2;
  ddpg   DDPG at the default config (normal noise), actor loop only.
For each: env-steps/s over the timed episodes (host clock, synchronised at both ends), ms per act() (it ends in a stream
synchronisation, so this is the call's full cost) and ms per step() (the call returns once its copies and kernels are
enqueued; their device time lands in the next act()), and the PCIe bytes per env step.  The card and its power limit are
read in the same run.

    python tools/host_env_timing.py [--rows ff rnn1 rnn2 ddpg] [--episodes 5] [--warmup 2]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

N, T, D, A = 1024, 128, 64, 8


class HostEnv:
    """Batched host env with pre-generated pinned dynamics (as bench.py's): the host side costs what a real env's output
    buffer costs, so the numbers isolate this side of the boundary.  Rewards are float64 when rew64 (as gym returns them)."""

    def __init__(self, N, D, A, T, seed=0, rew64=False):
        self.N, self.D, self.A, self.T = N, D, A, T
        rng = np.random.default_rng(seed)
        self._obs = torch.empty(T + 1, N, D, dtype=torch.float32, pin_memory=True)
        self._obs.numpy()[...] = rng.standard_normal((T + 1, N, D)).astype(np.float32)
        dt = torch.float64 if rew64 else torch.float32
        self._rew = torch.empty(T, N, dtype=dt, pin_memory=True)
        self._rew.numpy()[...] = rng.standard_normal((T, N))
        self._done = torch.zeros(T, N, dtype=torch.float32).pin_memory()
        self._done[T - 1] = 1.0                                   # episodes of T steps
        self._o = [self._obs[t].numpy() for t in range(T + 1)]
        self._r = [self._rew[t].numpy() for t in range(T)]
        self._d = [self._done[t].numpy() for t in range(T)]
        self.t = 0

    def reset(self):
        self.t = 0
        return {'low_dim': {'flat_inputs': self._o[0]}}, {}

    def step(self, action):
        t = self.t
        self.t = (t + 1) % self.T
        nxt = self._o[t + 1]
        return {'low_dim': {'flat_inputs': nxt}}, self._r[t], self._d[t], {'obs_next': nxt}


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'unknown'
    return name, pl


def _configs(kind, layers=1):
    from surreal_b200.session import Config
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    if kind == 'ddpg':
        from surreal_b200.main.ddpg_configs import DDPG_DEFAULT_LEARNER_CONFIG as LC, DDPG_DEFAULT_ENV_CONFIG as EC, \
            DDPG_DEFAULT_SESSION_CONFIG as SC
    else:
        from surreal_b200.main.ppo_configs import PPO_DEFAULT_LEARNER_CONFIG as LC, PPO_DEFAULT_ENV_CONFIG as EC, \
            PPO_DEFAULT_SESSION_CONFIG as SC
    lc, ec, sc = (Config(copy.deepcopy(c.to_dict())) for c in (LC, EC, SC))
    sc.folder = tempfile.mkdtemp(prefix='sb200_host_env_')
    make_synthetic_env_config(ec, N, D, A, seed=0)
    ec.limit_episode_length = T
    if kind == 'ff':                                              # bench.py's build_configs (BASELINE configs[1])
        lc.model.actor_fc_hidden_sizes = [256, 256]
        lc.model.critic_fc_hidden_sizes = [256, 256]
        lc.algo.ppo_mode = 'clip'
        lc.algo.rnn.if_rnn_policy = False
        lc.algo.n_step = lc.algo.stride = T
        lc.replay.batch_size = N
        lc.replay.memory_size = 2 * N
        lc.parameter_publish.exp_interval = N
        lc.parameter_publish.min_publish_interval = 0.0
        sc.agent.fetch_parameter_interval = T
    elif kind == 'rnn':
        lc.algo.rnn.rnn_layer = layers
    else:
        ec.num_agents = N
    return lc, ec, sc


def _bytes(kind, layers, H):
    """PCIe bytes per env step of the loop: observation, reward and done up (DDPG: also the action; its reward is float64),
    action and pd down (RNN: also the cells before the step, h and c of every layer)."""
    if kind == 'ddpg':
        return N * D * 4 + N * A * 4 + N * 8 + N * 4, N * A * 4
    h2d, d2h = N * D * 4 + 2 * N * 4, N * 3 * A * 4
    if kind == 'rnn':
        d2h += 2 * layers * N * H * 4
    return h2d, d2h


def run(kind, layers, episodes, warmup):
    from surreal_b200.launch import SurrealDefaultLauncher
    from surreal_b200.agent import PPOAgent, DDPGAgent
    from surreal_b200.learner import PPOLearner, DDPGLearner
    from surreal_b200.replay import FIFOReplay, UniformReplay
    lc, ec, sc = _configs(kind, layers)
    if kind == 'ddpg':
        la = SurrealDefaultLauncher(DDPGAgent, DDPGLearner, UniformReplay, sc, ec, lc)
    else:
        la = SurrealDefaultLauncher(PPOAgent, PPOLearner, FIFOReplay, sc, ec, lc)
    agent, replay, learner = la.setup_engine(env=HostEnv(N, D, A, T, rew64=(kind == 'ddpg')))
    w = agent.env
    assert w.host_env
    t_act, t_step = [0.0], [0.0]

    def episode():
        obs, _ = w.reset()
        for _ in range(T):
            t0 = time.perf_counter()
            a = agent.act(obs)
            t1 = time.perf_counter()
            obs, _, _, _ = w.step(a)
            t_act[0] += t1 - t0
            t_step[0] += time.perf_counter() - t1
        if kind == 'ff':
            learner.main_loop()                                   # FIFO -> learn -> publish, as bench.py's e2e row

    for _ in range(warmup):
        episode()
    torch.cuda.synchronize()
    t_act[0] = t_step[0] = 0.0
    t0 = time.perf_counter()
    for _ in range(episodes):
        episode()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    H = lc.algo.rnn.rnn_hidden if kind == 'rnn' else 0
    h2d, d2h = _bytes(kind, layers, H)
    res = dict(row=kind + (str(layers) if kind == 'rnn' else ''), env_steps_per_s=round(N * T * episodes / dt),
               ms_per_episode=round(dt / episodes * 1e3, 3), ms_per_act=round(t_act[0] / (episodes * T) * 1e3, 4),
               ms_per_step=round(t_step[0] / (episodes * T) * 1e3, 4), h2d_bytes_per_step=h2d, d2h_bytes_per_step=d2h,
               actors=N, obs_dim=D, act_dim=A, horizon=T, learner=(kind == 'ff'))
    if kind == 'rnn':
        res.update(rnn_hidden=H, rnn_layer=layers)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', nargs='+', default=['ff', 'rnn1', 'rnn2', 'ddpg'])
    ap.add_argument('--episodes', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('host_env_timing needs a CUDA device')
    name, pl = _card()
    print('card: %s, power limit: %s' % (name, pl))
    for row in args.rows:
        kind, layers = ('rnn', int(row[3:])) if row.startswith('rnn') else (row, 1)
        res = run(kind, layers, args.episodes, args.warmup)
        res.update(card=name, power_limit=pl)
        print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()

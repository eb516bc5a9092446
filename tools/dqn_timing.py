#!/usr/bin/env python
"""Timing of single-GPU DQN training (64-dim observations, 18 discrete actions, dueling 256-256 towers with double Q,
1 M-slot replay pre-filled, batch 4096, 1024 actors on the discrete synthetic env), one process, arms alternated, every
window after warm-up and ending in a device synchronise:

  learner   updates/s of learn(sample()) -- host index stream, one graph per update -- against
            learn_from_replay(K) -- device sampler, K updates per graph -- for K in 1, 8, 32;
  engine    ReplayEngine env-steps/s and updates/s at T = 32 for K in 32, 8, on UniformReplay and PrioritizedReplay.
The card's name and power limit are read in the same run.

    python tools/dqn_timing.py [--rounds 3] [--out dqn_timing.json]
"""
import argparse
import copy
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

D, NA, B, CAP, N = 64, 18, 4096, 1 << 20, 1024


def configs(prioritized=False):
    from surreal_b200.session import Config
    from surreal_b200.main.dqn_configs import (DQN_DEFAULT_LEARNER_CONFIG, DQN_DEFAULT_ENV_CONFIG,
                                               DQN_DEFAULT_SESSION_CONFIG, make_discrete_synthetic_env_config)
    lc = Config(copy.deepcopy(DQN_DEFAULT_LEARNER_CONFIG.to_dict()))
    ec = Config(copy.deepcopy(DQN_DEFAULT_ENV_CONFIG.to_dict()))
    sc = Config(copy.deepcopy(DQN_DEFAULT_SESSION_CONFIG.to_dict()))
    sc.folder = tempfile.mkdtemp()
    make_discrete_synthetic_env_config(ec, N, D, NA, seed=1)
    ec.num_agents, ec.limit_episode_length = N, 200
    lc.model.convs, lc.model.fc_hidden_sizes, lc.model.dueling = [], [256, 256], True
    lc.algo.target_network_update_freq, lc.algo.exploration.steps = 40000, 100000
    lc.algo.prioritized.enabled = prioritized
    lc.eval.eps = 0.05
    lc.replay.batch_size, lc.replay.memory_size, lc.replay.sampling_start_size = B, CAP, 3000
    return lc, ec, sc


def prefill(R):
    g = torch.Generator(device='cuda').manual_seed(4)
    R.r_obs.normal_(generator=g)
    R.r_obs_next.normal_(generator=g)
    R.r_act.copy_(torch.randint(0, NA, R.r_act.shape, device='cuda', generator=g).float())
    R.r_rew.normal_(generator=g)
    R.r_done.copy_((torch.rand(CAP, device='cuda', generator=g) < 0.005).float())
    R.state[0], R.state[1], R.state[3] = 0, CAP, CAP
    R.mark_device_inserts()
    R.snapshot_view(0)


def quiet(L):
    L.tensorplex.add_scalars = lambda *a, **k: None
    L.periodic_checkpoint = lambda *a, **k: None
    return L


def wall(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def spread(v):
    return {'median': float(np.median(v)), 'min': float(np.min(v)), 'max': float(np.max(v))}


def learner_leg(rounds):
    from surreal_b200.learner import DQNLearner
    from surreal_b200.replay import UniformReplay
    lc, ec, sc = configs()
    R = UniformReplay(lc, ec, sc)
    prefill(R)
    random.seed(5)
    arms = {'learn(sample())': (quiet(DQNLearner(lc, ec, sc)), 1)}
    for K in (1, 8, 32):
        arms['learn_from_replay(K=%d)' % K] = (quiet(DQNLearner(lc, ec, sc)), K)
    fns = {}
    for name, (L, K) in arms.items():
        fns[name] = (lambda L=L: L.learn(R.sample(B, out=L.replay_out_buffers()))) if name.startswith('learn(') else \
            (lambda L=L, K=K: L.learn_from_replay(R, K))
        for _ in range(3):
            fns[name]()
    rate = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (L, K) in arms.items():
            calls = max(1, 256 // K)
            rate[name].append(calls * K / wall(fns[name], calls))
    return {k: dict(updates_per_s=spread(v), all=v) for k, v in rate.items()}


def engine_leg(rounds, steps):
    from surreal_b200.launch import SurrealDefaultLauncher, ReplayEngine
    from surreal_b200.agent import QAgent
    from surreal_b200.learner import DQNLearner
    from surreal_b200.replay import UniformReplay, PrioritizedReplay
    res = {}
    T = 32
    for K in (32, 8):
        engines = {}
        for per in (False, True):
            lc, ec, sc = configs(per)
            la = SurrealDefaultLauncher(QAgent, DQNLearner, PrioritizedReplay if per else UniformReplay, sc, ec, lc)
            agent, replay, learner = la.setup_engine()
            quiet(learner)
            prefill(replay)
            eng = ReplayEngine(agent, replay, learner, T, K)
            eng.prime()
            for _ in range(3):
                eng.step()
            eng.drain()
            engines['prioritized' if per else 'uniform'] = eng
        secs = {k: [] for k in engines}
        for _ in range(rounds):
            for name, eng in engines.items():
                secs[name].append(wall(eng.step, steps) / steps)
        res['T%d_K%d' % (T, K)] = {k: {'step_ms': spread([1e3 * s for s in v]),
                                       'env_steps_per_s': spread([N * T / s for s in v]),
                                       'updates_per_s': spread([K / s for s in v])} for k, v in secs.items()}
        del engines
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--engine-steps', type=int, default=30)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs the GPU'
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    res = {'card': torch.cuda.get_device_name(0), 'nvidia_smi': smi}
    res['learner'] = learner_leg(args.rounds)
    print(json.dumps(res['learner']), flush=True)
    res['engine'] = engine_leg(args.rounds, args.engine_steps)
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as fp:
            json.dump(res, fp, indent=1)


if __name__ == '__main__':
    main()

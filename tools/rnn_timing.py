#!/usr/bin/env python
"""RNN-mode timings at the default PPO config (64 windows of n_step 25, horizon 5, LSTM(100), heads 300-200) for 1, 2 and 3
LSTM layers: one learn() as a CUDA graph and eagerly, and one act() step of 1024 device actors.  CUDA events after a
warm-up; prints the card, its power limit and one JSON line per depth.

    python tools/rnn_timing.py [--layers 1 2 3] [--iters 20] [--warmup 5] [--actors 1024]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'unknown'
    return name, pl


def _configs(layers, N, D, A):
    from surreal_b200.session import Config
    from surreal_b200.main.ppo_configs import (PPO_DEFAULT_LEARNER_CONFIG, PPO_DEFAULT_ENV_CONFIG, PPO_DEFAULT_SESSION_CONFIG,
                                               make_synthetic_env_config)
    lc = Config(copy.deepcopy(PPO_DEFAULT_LEARNER_CONFIG.to_dict()))
    ec = Config(copy.deepcopy(PPO_DEFAULT_ENV_CONFIG.to_dict()))
    sc = Config(copy.deepcopy(PPO_DEFAULT_SESSION_CONFIG.to_dict()))
    sc.folder = tempfile.mkdtemp()
    lc.algo.rnn.rnn_layer = layers
    make_synthetic_env_config(ec, N, D, A, seed=0)
    return lc, ec, sc


def _batch(lc, D, A, layers, rng):
    B, n, H = lc.replay.batch_size, lc.algo.n_step, lc.algo.rnn.rnn_hidden
    pd = np.concatenate([np.tanh(rng.standard_normal((B, n, A))) * 0.5, np.full((B, n, A), 0.4)], -1).astype(np.float32)
    return {'obs': {'low_dim': {'flat_inputs': rng.standard_normal((B, n, D)).astype(np.float32)}},
            'obs_next': {'low_dim': {'flat_inputs': rng.standard_normal((B, 1, D)).astype(np.float32)}},
            'actions': np.clip(rng.standard_normal((B, n, A)) * 0.4, -1, 1), 'rewards': rng.standard_normal((B, n)) * 0.3,
            'dones': np.zeros((B, n), np.float32), 'persistent_infos': [pd],
            'onetime_infos': [(rng.standard_normal((B, layers, H)) * 0.2).astype(np.float32),
                              (rng.standard_normal((B, layers, H)) * 0.2).astype(np.float32)]}


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), float(np.min(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--layers', type=int, nargs='+', default=[1, 2, 3])
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--actors', type=int, default=1024)
    args = ap.parse_args()
    from surreal_b200.learner import PPOLearner
    from surreal_b200.agent import PPOAgent
    name, pl = _card()
    print('card: %s, power limit: %s' % (name, pl))
    D, A = 17, 6
    for layers in args.layers:
        res = dict(layers=layers)
        rng = np.random.default_rng(layers)
        for graph in (True, False):
            lc, ec, sc = _configs(layers, args.actors, D, A)
            L = PPOLearner(lc, ec, sc)
            L.use_cuda_graph = graph
            batch = _batch(lc, D, A, layers, rng)
            med, best = _time(lambda: L.learn(batch), args.iters, args.warmup)
            res['learn_ms_graph' if graph else 'learn_ms_eager'] = round(med, 3)
            res['learn_ms_graph_min' if graph else 'learn_ms_eager_min'] = round(best, 3)
            del L
        lc, ec, sc = _configs(layers, args.actors, D, A)
        ag = PPOAgent(lc, ec, sc, 0, 'training')
        obs = torch.randn(args.actors, D, device='cuda')
        med, best = _time(lambda: ag.act(obs), args.iters * 5, args.warmup)
        res['act_ms'], res['act_ms_min'] = round(med, 4), round(best, 4)
        res.update(B=lc.replay.batch_size, n_step=lc.algo.n_step, horizon=lc.algo.rnn.horizon, H=lc.algo.rnn.rnn_hidden,
                   actors=args.actors, card=name, power_limit=pl)
        print(json.dumps(res))


if __name__ == '__main__':
    main()

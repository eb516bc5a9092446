#!/usr/bin/env python
"""CNN + LSTM timings at the default PPO config (64 windows of n_step 25, horizon 5, cnn_feature_dim 256, LSTM(100), heads
300-200) on [4, 84, 84] uint8 frames: one learn() as a CUDA graph and eagerly (device batch), and one act() step of 256
and 1024 actors with device frames and with host (numpy) frames.  CUDA events after a warm-up; prints the card, its power
limit and one JSON line.

    python tools/pixel_rnn_timing.py [--iters 20] [--warmup 5] [--actors 256 1024]
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

FRAME, A = (4, 84, 84), 6


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'unknown'
    return name, pl


def _configs(N):
    """PPO_DEFAULT_LEARNER_CONFIG unmodified except use_z_filter (the reference refuses it without low-dim input)."""
    from surreal_b200.session import Config
    from surreal_b200.main.ppo_configs import (PPO_DEFAULT_LEARNER_CONFIG, PPO_DEFAULT_ENV_CONFIG, PPO_DEFAULT_SESSION_CONFIG,
                                               make_synthetic_pixel_env_config)
    lc = Config(copy.deepcopy(PPO_DEFAULT_LEARNER_CONFIG.to_dict()))
    ec = Config(copy.deepcopy(PPO_DEFAULT_ENV_CONFIG.to_dict()))
    sc = Config(copy.deepcopy(PPO_DEFAULT_SESSION_CONFIG.to_dict()))
    sc.folder = tempfile.mkdtemp()
    lc.algo.use_z_filter = False
    make_synthetic_pixel_env_config(ec, N, frame_shape=FRAME, action_dim=A)
    return lc, ec, sc


def _batch(lc, rng):
    """A device batch: frames, actions, behaviour policy and the windows' initial cells as CUDA tensors."""
    B, n, H, Lr = lc.replay.batch_size, lc.algo.n_step, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer
    d = lambda a: torch.as_tensor(a).cuda()  # noqa: E731
    pd = np.concatenate([np.tanh(rng.standard_normal((B, n, A))) * 0.5, np.full((B, n, A), 0.4)], -1).astype(np.float32)
    return {'obs': {'pixel': {'camera0': d(rng.integers(0, 256, (B, n) + FRAME, dtype=np.uint8))}},
            'obs_next': {'pixel': {'camera0': d(rng.integers(0, 256, (B, 1) + FRAME, dtype=np.uint8))}},
            'actions': d(np.clip(rng.standard_normal((B, n, A)) * 0.4, -1, 1).astype(np.float32)),
            'rewards': d((rng.standard_normal((B, n)) * 0.3).astype(np.float32)), 'dones': d(np.zeros((B, n), np.float32)),
            'persistent_infos': [d(pd)],
            'onetime_infos': [d((rng.standard_normal((B, Lr, H)) * 0.2).astype(np.float32)),
                              d((rng.standard_normal((B, Lr, H)) * 0.2).astype(np.float32))]}


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
    return round(float(np.median(ms)), 4), round(float(np.min(ms)), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--actors', type=int, nargs='+', default=[256, 1024])
    args = ap.parse_args()
    from surreal_b200.learner import PPOLearner
    from surreal_b200.agent import PPOAgent
    name, pl = _card()
    print('card: %s, power limit: %s' % (name, pl))
    rng = np.random.default_rng(0)
    lc, _, _ = _configs(1)
    res = dict(B=lc.replay.batch_size, n_step=lc.algo.n_step, horizon=lc.algo.rnn.horizon, H=lc.algo.rnn.rnn_hidden,
               cnn_feature_dim=lc.model.cnn_feature_dim, frame=list(FRAME), card=name, power_limit=pl)
    batch = _batch(lc, rng)
    for graph in (True, False):
        L = PPOLearner(*_configs(1))
        L.use_cuda_graph = graph
        res['learn_ms_graph' if graph else 'learn_ms_eager'], res['learn_ms_graph_min' if graph else 'learn_ms_eager_min'] = \
            _time(lambda: L.learn(batch), args.iters, args.warmup)
        del L
    for N in args.actors:
        ag = PPOAgent(*_configs(N), 0, 'training')
        dev = torch.randint(0, 256, (N,) + FRAME, dtype=torch.uint8, device='cuda')
        host = dev.cpu().numpy()
        res['act_ms_device_%d' % N], _ = _time(lambda: ag.act({'pixel': {'camera0': dev}}), args.iters * 5, args.warmup)
        res['act_ms_host_%d' % N], _ = _time(lambda: ag.act({'pixel': {'camera0': host}}), args.iters * 5, args.warmup)
        del ag
    print(json.dumps(res))


if __name__ == '__main__':
    main()

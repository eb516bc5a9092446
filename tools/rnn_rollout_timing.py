#!/usr/bin/env python
"""Device-env rollout chunks of the recurrent PPO policy at the default config (D 64, LSTM(100), head 300-200, A 8) for 1 and
2 LSTM layers and several actor counts, n_step = stride = T: ms per chunk through agent.main_loop (CUDA-graph replay) on
the persistent kernel (sb200_ppo_rollout_rnn_f32) and on the per-step launch chain, the two alternated in one process.
Prints the card, its power limit and one JSON line per (layers, N).

    python tools/rnn_rollout_timing.py [--layers 1 2] [--actors 256 1024 4096] [--T 32] [--reps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = 'unknown'
    return name, pl


def _agent(layers, N, T):
    from helpers import ppo_configs
    from surreal_b200.agent import PPOAgent
    from surreal_b200.env import SyntheticEnv
    from surreal_b200.replay import FIFOReplay
    D, A, H = 64, 8, 100
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=(300, 200), critic_h=(300, 200), n_step=T, stride=T, B=N,
                             memory_size=4 * N)
    lc.algo.rnn.if_rnn_policy = True
    lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = 5, H, layers
    ec.num_envs = N
    replay = FIFOReplay(lc, ec, sc)
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    env = SyntheticEnv(N, D, A, limit_episode_length=200, seed=1)
    ag.env = w = ag.prepare_env_agent(env)
    ag._obs, _ = w.reset()
    return ag, replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--layers', type=int, nargs='+', default=[1, 2])
    ap.add_argument('--actors', type=int, nargs='+', default=[256, 1024, 4096])
    ap.add_argument('--T', type=int, default=32)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('rnn_rollout_timing needs a CUDA device')
    from surreal_b200.ops import graphs_enabled
    assert graphs_enabled()
    name, pl = _card()
    print('card: %s, power limit %s' % (name, pl))
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    T = args.T
    for layers in args.layers:
        for N in args.actors:
            paths = {}
            for path in ('persistent', 'chain'):
                ag, replay = _agent(layers, N, T)
                if path == 'chain':
                    ag.env.persistent_rollout = False
                assert ag.rollout_chunk_supported() == (path == 'persistent')
                paths[path] = (ag, replay)
            fp = paths['persistent'][0].rollout_footprint()
            ms = {p: [] for p in paths}
            for rep in range(args.warmup + args.reps):
                for p, (ag, replay) in paths.items():          # alternated, so that both see the same machine state
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    ag.main_loop(max_steps=T)
                    e1.record()
                    torch.cuda.synchronize()
                    if rep >= args.warmup:
                        ms[p].append(e0.elapsed_time(e1))
            med = {p: float(np.median(v)) for p, v in ms.items()}
            ctas = (N + 7) // 8
            print(json.dumps(dict(layers=layers, N=N, T=T, ctas=ctas, sms=n_sm, one_wave=ctas <= n_sm, footprint=fp,
                                  persistent_ms=round(med['persistent'], 4), chain_ms=round(med['chain'], 4),
                                  speedup=round(med['chain'] / med['persistent'], 2),
                                  persistent_env_steps_per_s=round(N * T / med['persistent'] * 1e3),
                                  chain_env_steps_per_s=round(N * T / med['chain'] * 1e3),
                                  spread_persistent=[round(min(ms['persistent']), 4), round(max(ms['persistent']), 4)],
                                  spread_chain=[round(min(ms['chain']), 4), round(max(ms['chain']), 4)],
                                  card=name, power_limit=pl)),
                  flush=True)
            del paths
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()

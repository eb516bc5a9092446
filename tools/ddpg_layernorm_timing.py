#!/usr/bin/env python
"""Timing of the LayerNorm DDPG networks (model.use_layernorm) against the plain ones, alternated in one process:

  learn   DDPGLearner.learn() ms at batch 4096, actor 300-200, critic 400-300 (64-dim observations, 8-dim actions),
          one CUDA graph per call; the same host batch every call;
  act     DDPGAgent.act() ms on 1024 actors with device observations, without and with adaptive parameter noise.
Each leg alternates off / on for `--rounds` rounds and reports the median.  The card's name and power limit are read
in the same run.

    python tools/ddpg_layernorm_timing.py [--rounds 5] [--reps 50] [--out ddpg_layernorm_timing.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

D, A = 64, 8


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def make_learner(ln, B=4096):
    from helpers import ddpg_configs
    from surreal_b200.learner import DDPGLearner
    lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=(300, 200), critic_h=(400, 300), B=B)
    lc.model.use_layernorm = ln
    L = DDPGLearner(lc, ec, sc)
    L.tensorplex.add_scalars = lambda *a, **k: None
    L.periodic_checkpoint = lambda *a, **k: None
    rng = np.random.default_rng(0)
    batch = {'obs': {'low_dim': {'flat_inputs': rng.standard_normal((B, D)).astype(np.float32)}},
             'obs_next': {'low_dim': {'flat_inputs': rng.standard_normal((B, D)).astype(np.float32)}},
             'actions': rng.uniform(-1, 1, (B, A)).astype(np.float32), 'rewards': rng.standard_normal((B, 1)),
             'dones': np.zeros((B, 1))}
    return lambda: L.learn(batch)


def make_agent(ln, param_noise, N=1024):
    from helpers import ddpg_configs
    from surreal_b200.agent import DDPGAgent
    lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=(300, 200), critic_h=(400, 300))
    lc.model.use_layernorm = ln
    lc.algo.exploration.param_noise_type = param_noise
    ec.num_envs, ec.num_agents = N, N
    ag = DDPGAgent(lc, ec, sc, 0, 'training')
    if param_noise is not None:
        ag.apply_param_noise()
    x = torch.randn(N, D, device='cuda')
    return lambda: ag.act(x)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs the GPU'
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    legs = {'learn_B4096': lambda ln: make_learner(ln), 'act_1024': lambda ln: make_agent(ln, None),
            'act_1024_param_noise': lambda ln: make_agent(ln, 'adaptive_normal')}
    res = {'card': torch.cuda.get_device_name(0), 'nvidia_smi': smi}
    for name, mk in legs.items():
        fns = {ln: mk(ln) for ln in (False, True)}
        t = {False: [], True: []}
        for _ in range(args.rounds):
            for ln in (False, True):
                t[ln].append(timed(fns[ln], args.reps))
        res[name] = {'off_ms': float(np.median(t[False])), 'on_ms': float(np.median(t[True])),
                     'off_all': t[False], 'on_all': t[True]}
        print(name, 'layernorm off %.4f ms  on %.4f ms' % (res[name]['off_ms'], res[name]['on_ms']), flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as fp:
            json.dump(res, fp, indent=1)


if __name__ == '__main__':
    main()

#!/usr/bin/env python
"""Timing of prioritized replay at BASELINE configs[2] size (64-dim observations, 8-dim actions, a 1 M-slot ring
pre-filled, batch 4096, actor 300-200, critic 400-300, 1024 actors on the synthetic env), one process:

  kernels   CUDA events over back-to-back launches of PrioritizedReplay's entries: admit of one chunk of inserts
            (1024 actors x 32 steps = 32768 slots) with its rebuild, sample + gather + weights at batch 4096, the priority
            update of a 4096 batch with its rebuild, and a full rebuild of every subtree;
  engine    ReplayEngine updates/s and env-steps/s with PrioritizedReplay against UniformReplay, two streams, for
            (T, K) in (32, 32), (32, 8), the arms alternated round by round.
The card's name and power limit are read in the same run.

    python tools/per_timing.py [--rounds 3] [--engine-steps 30] [--out per_timing.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from ddpg_engine_timing import A, B, CAP, D, N, configs, events_ms, prefill, quiet, wall  # noqa: E402

CHUNK = N * 32


def kernel_leg():
    from surreal_b200.replay import PrioritizedReplay
    lc, ec, sc = configs()
    R = PrioritizedReplay(lc, ec, sc)
    R.state[3] = CAP
    prefill(R)                                                 # full ring, every slot admitted
    rng = torch.Generator(device='cuda').manual_seed(3)
    idx = torch.randint(0, CAP, (B,), device='cuda', generator=rng)
    prio = torch.rand(B, device='cuda', generator=rng) + 1e-3
    f = lambda w: torch.empty(B, w, device='cuda')  # noqa: E731
    out = dict(obs=f(D), obs_next=f(D), actions=f(A), rewards=f(1), dones=f(1))

    def admit_chunk():
        R.state[3] += CHUNK                                   # one chunk of inserts, as the SSAR step counts them
        R.admit()
    return {'admit_32768_ms': events_ms(admit_chunk, 100),
            'sample_gather_weights_b4096_ms': events_ms(lambda: R.sample_device(B, out=out), 200),
            'update_b4096_ms': events_ms(lambda: R.update_priorities_device(idx, prio), 200),
            'full_rebuild_ms': events_ms(lambda: R.rebuild(full=True), 100),
            'uniform_sample_gather_b4096_ms': events_ms(lambda: super(PrioritizedReplay, R).sample_device(B, out=out),
                                                         200)}


def engine_leg(rounds, steps):
    from surreal_b200.launch import SurrealDefaultLauncher, ReplayEngine
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.learner import DDPGLearner
    from surreal_b200.replay import UniformReplay, PrioritizedReplay
    res = {}
    for T, K in ((32, 32), (32, 8)):
        engines = {}
        for name, cls in (('prioritized', PrioritizedReplay), ('uniform', UniformReplay)):
            lc, ec, sc = configs()
            la = SurrealDefaultLauncher(DDPGAgent, DDPGLearner, cls, sc, ec, lc)
            agent, replay, learner = la.setup_engine()
            quiet(learner)
            replay.state[3] = CAP
            prefill(replay)
            eng = ReplayEngine(agent, replay, learner, T, K)
            eng.prime()
            for _ in range(3):
                eng.step()
            eng.drain()
            engines[name] = eng
        secs = {k: [] for k in engines}
        for _ in range(rounds):
            for name, eng in engines.items():
                secs[name].append(wall(eng.step, steps) / steps)
        res['T%d_K%d' % (T, K)] = {k: {'step_ms': 1e3 * float(np.median(v)), 'env_steps_per_s': N * T / float(np.median(v)),
                                       'updates_per_s': K / float(np.median(v)), 'all_step_s': v} for k, v in secs.items()}
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
    res['kernels'] = kernel_leg()
    print(json.dumps(res['kernels']), flush=True)
    res['engine'] = engine_leg(args.rounds, args.engine_steps)
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as fp:
            json.dump(res, fp, indent=1)


if __name__ == '__main__':
    main()

#!/usr/bin/env python
"""Learning curves and env-step timing of the classic-control tasks (surreal_b200.env.classic), one process:

  train   each learning case of tests/classic_learning.py (the configs the learning tests commit): mean first-episode
          return of 64 fresh eval actors against env steps and training wall time (evaluations excluded);
  env     the env step (sb200_env_step_f32) of CartPole-v1 and Pendulum-v1 at 1024, 16 384 and 65 536 actors beside
          the synthetic env's (64-dim state, 8-dim action): CUDA events around replays of a graph
          of 100 steps after warm-up, cycling through 16 random action sets.
The card's name, power limit and maximum SM clock are read in the same run.

    python tools/classic_control_train.py train [--cases ppo_cartpole_mlp,...] [--iterations 300] [--max-seconds 60]
    python tools/classic_control_train.py env [--reps 2000]
    [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def card():
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True)
    return smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else torch.cuda.get_device_name(0)


def train(args):
    import classic_learning as CL
    out = {}
    names = args.cases.split(',') if args.cases else list(CL.CASES)
    for name in names:
        case = CL.CASES[name]
        print('== %s (%s)' % (name, case.env), flush=True)
        print('%12s %10s %12s' % ('env steps', 'seconds', 'return'), flush=True)
        _, curve = CL.train(case, args.iterations, eval_every=args.eval_every, max_seconds=args.max_seconds,
                            log=lambda n, st, sec, ret: print('%12d %10.1f %12.1f' % (st, sec, ret), flush=True))
        out[name] = {'env': case.env, 'bar': case.bar, 'curve': curve}
    return out


def env_timing(args):
    from surreal_b200.env import CartPoleEnv, PendulumEnv, SyntheticEnv
    rows = []
    for N in (1024, 16384, 65536):
        envs = [('CartPole-v1', CartPoleEnv(N, seed=1)), ('Pendulum-v1', PendulumEnv(N, seed=1)),
                ('synthetic D=64 A=8', SyntheticEnv(N, 64, 8, seed=1))]
        for name, env in envs:
            env.reset()
            gen = torch.Generator(device='cuda').manual_seed(0)
            if name == 'CartPole-v1':
                acts = torch.nn.functional.one_hot(torch.randint(0, 2, (16, N), device='cuda', generator=gen), 2).float()
            else:
                acts = torch.rand(16, N, env.A, device='cuda', generator=gen) * 2 - 1
            acts = [a.contiguous() for a in acts]
            for k in range(50):
                env.step(acts[k % 16])
            # the steps are replayed from a CUDA graph, so the window holds kernel time and not the host's launch rate
            torch.cuda.synchronize()
            g, st = torch.cuda.CUDAGraph(), torch.cuda.Stream()
            st.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(st), torch.cuda.graph(g):
                for k in range(100):
                    env.step(acts[k % 16])
            torch.cuda.current_stream().wait_stream(st)
            g.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps // 100):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            steps = 100 * (args.reps // 100)
            us = 1000.0 * e0.elapsed_time(e1) / steps
            rows.append({'env': name, 'N': N, 'us_per_step': us, 'actor_steps_per_s': N / us * 1e6})
            print('%-20s N=%6d  %8.2f us/step  %10.3g actor steps/s' % (name, N, us, N / us * 1e6), flush=True)
    return rows


def main():
    p = argparse.ArgumentParser()
    p.add_argument('mode', choices=['train', 'env'])
    p.add_argument('--cases', default='')
    p.add_argument('--iterations', type=int, default=300)
    p.add_argument('--eval-every', type=int, default=10)
    p.add_argument('--max-seconds', type=float, default=None)
    p.add_argument('--reps', type=int, default=2000)
    p.add_argument('--out', default=None)
    args = p.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    info = card()
    print('card:', info, flush=True)
    res = {'card': info, args.mode: train(args) if args.mode == 'train' else env_timing(args)}
    if args.out:
        with open(args.out, 'w') as fp:
            json.dump(res, fp, indent=1)


if __name__ == '__main__':
    main()

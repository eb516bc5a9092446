#!/usr/bin/env python
"""Timing of single-GPU DDPG training at BASELINE configs[2] size (64-dim observations, 8-dim actions, 1 M-slot
UniformReplay pre-filled, batch 4096, actor 300-200, critic 400-300, 1024 actors on the synthetic env), one process,
arms alternated, every window after warm-up and ending in a device synchronise:

  learner   updates/s of learn(sample()) -- host index stream, one graph per update -- against
            learn_from_replay(K) -- device sampler, K updates per graph -- for K in 1, 8, 32;
  sampler   sb200_uniform_sample_gather_f32 alone (CUDA events) at batch 4096 and 2^20: ms and GB/s on 2*552+8 bytes per
            sample, beside gather_multi_kernel on indices made beforehand and a device-to-device copy of 1 GiB
            (read + write bytes) as the measured copy peak.  Launches run back to back: the ring (579 MB) does not fit
            in L2, the batch-4096 outputs do;
  engine    ReplayEngine env-steps/s and updates/s on two streams against the one-stream schedule (overlap=False), for
            (T, K) in (32, 32), (32, 8).
The card's name and power limit are read in the same run.

    python tools/ddpg_engine_timing.py [--rounds 3] [--out ddpg_engine_timing.json]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

D, A, B, CAP, N = 64, 8, 4096, 1 << 20, 1024
REC_BYTES = (2 * D + A + 2) * 4


def configs():
    from helpers import ddpg_configs
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=(300, 200), critic_h=(400, 300), B=B, n_step=3, memory_size=CAP, start=3000)
    make_synthetic_env_config(ec, N, D, A, seed=1)
    ec.num_agents = N
    return lc, ec, sc


def prefill(R):
    g = torch.Generator(device='cuda').manual_seed(4)
    R.r_obs.normal_(generator=g)
    R.r_obs_next.normal_(generator=g)
    R.r_act.uniform_(-1, 1, generator=g)
    R.r_rew.normal_(generator=g)
    R.r_done.copy_((torch.rand(CAP, device='cuda', generator=g) < 0.005).float())
    R.state[0], R.state[1] = 0, CAP
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


def events_ms(fn, reps):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def learner_leg(rounds):
    from surreal_b200.learner import DDPGLearner
    from surreal_b200.replay import UniformReplay
    lc, ec, sc = configs()
    R = UniformReplay(lc, ec, sc)
    prefill(R)
    random.seed(5)
    arms = {'learn(sample())': (quiet(DDPGLearner(lc, ec, sc)), 1)}
    for K in (1, 8, 32):
        arms['learn_from_replay(K=%d)' % K] = (quiet(DDPGLearner(lc, ec, sc)), K)
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
    return {k: {'updates_per_s': float(np.median(v)), 'all': v} for k, v in rate.items()}


def sampler_leg():
    from surreal_b200.replay import UniformReplay
    from surreal_b200.replay.base import gather_fields
    lc, ec, sc = configs()
    R = UniformReplay(lc, ec, sc)
    prefill(R)
    src, dst = torch.empty(1 << 28, device='cuda'), torch.empty(1 << 28, device='cuda')
    copy_gbs = 2 * src.numel() * 4 / (events_ms(lambda: dst.copy_(src), 10) / 1e3) / 1e9
    del src, dst
    out = {'bytes_per_sample': 2 * REC_BYTES + 8, 'copy_peak_gbs_measured': copy_gbs}
    for batch in (B, 1 << 20):
        f = lambda w: torch.empty(batch, w, device='cuda')  # noqa: E731
        o = dict(obs=f(D), obs_next=f(D), actions=f(A), rewards=f(1), dones=f(1))
        idx = torch.randint(0, CAP, (batch,), device='cuda', dtype=torch.int64)
        pairs = [(R.r_obs, o['obs'], D), (R.r_obs_next, o['obs_next'], D), (R.r_act, o['actions'], A),
                 (R.r_rew, o['rewards'], 1), (R.r_done, o['dones'], 1)]
        R.sample_device(batch, out=o)
        reps = 200 if batch == B else 20
        ms_s = events_ms(lambda: R.sample_device(batch, out=o), reps)
        ms_g = events_ms(lambda: gather_fields(pairs, None, idx, batch), reps)
        gbs = lambda ms: batch * (2 * REC_BYTES + 8) / (ms / 1e3) / 1e9  # noqa: E731
        out['batch_%d' % batch] = {'sample_gather_ms': ms_s, 'sample_gather_gbs': gbs(ms_s),
                                   'sample_gather_frac_of_copy_peak': gbs(ms_s) / copy_gbs,
                                   'gather_multi_ms': ms_g, 'gather_multi_gbs': gbs(ms_g)}
    return out


def engine_leg(rounds, steps):
    from surreal_b200.launch import SurrealDefaultLauncher, ReplayEngine
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.learner import DDPGLearner
    from surreal_b200.replay import UniformReplay
    res = {}
    for T, K in ((32, 32), (32, 8)):
        engines = {}
        for overlap in (True, False):
            lc, ec, sc = configs()
            la = SurrealDefaultLauncher(DDPGAgent, DDPGLearner, UniformReplay, sc, ec, lc)
            agent, replay, learner = la.setup_engine()
            quiet(learner)
            prefill(replay)
            eng = ReplayEngine(agent, replay, learner, T, K, overlap=overlap)
            eng.prime()
            for _ in range(3):
                eng.step()
            eng.drain()
            engines['two_streams' if overlap else 'one_stream'] = eng
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
    res['learner'] = learner_leg(args.rounds)
    print(json.dumps(res['learner']), flush=True)
    res['sampler'] = sampler_leg()
    print(json.dumps(res['sampler']), flush=True)
    res['engine'] = engine_leg(args.rounds, args.engine_steps)
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as fp:
            json.dump(res, fp, indent=1)


if __name__ == '__main__':
    main()

#!/usr/bin/env python
"""Timing of DDPG parameter-space noise on the default actor (64-300-200-8, 81 308 parameters):

  forward   sb200_mlp_forward_per_actor_f32 at N = 256 / 1024 / 4096 actors, normal and adaptive at a distance step
            (CUDA events over many launches); achieved bytes/s = N * flat actor bytes / kernel time (weights only:
            observations and outputs are under 1 % of the bytes), against the 3.35 TB/s HBM3 data-sheet figure;
  apply     sb200_ddpg_param_noise_apply_f32 per fetch (CUDA events), bytes written = N * stride * 4;
  act       DDPGAgent.act() ms with and without parameter noise: host-env loop (numpy in / numpy out, one sync per call)
            and device-env chunk (main_loop of SyntheticEnv as one CUDA graph), 1024 actors.
The card's name and power limit are read in the same run.

    python tools/param_noise_timing.py [--reps 200] [--out param_noise_timing.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))

D, A, HID = 64, 8, (300, 200)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def events(fn, reps):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps            # ms per launch


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                          # noqa: BLE001
        q = 'nvidia-smi unavailable: %s' % e
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q)


def kernels(reps):
    from surreal_b200 import ops, _lib
    from surreal_b200.agent.ddpg_agent import param_noise_stride
    dev = torch.device('cuda', 0)
    dims = [D, *HID, A]
    net = ops.FlatNet(dims, [ops.ACT_RELU, ops.ACT_RELU, ops.ACT_TANH], dev)
    net.params.normal_(0, 0.05)
    stride = param_noise_stride(net.size)
    L = _lib.lib()
    rows = []
    for N in (256, 1024, 4096):
        images = torch.zeros(N * stride, device=dev)
        sigma = torch.full((N,), 0.05, dtype=torch.float64, device=dev)
        x = torch.randn(N, D, device=dev)
        out = torch.empty(N, A, device=dev)
        dist = torch.zeros(N, device=dev)
        state = torch.zeros(2, dtype=torch.int64, device=dev)
        d, dimg = net.desc(), net.desc(images)
        st = ops._stream()
        ms_apply = events(lambda: L.sb200_ddpg_param_noise_apply_f32(C.byref(d), N, _p(images), stride, _p(sigma), None,
                                                                     5, 0, None, None, 1.15, 0.005, st), reps)
        ms_fwd = events(lambda: L.sb200_mlp_forward_per_actor_f32(C.byref(dimg), stride, _p(x), D, N, _p(out), A, None,
                                                                  None, 10, None, st), reps)

        def adaptive():                               # every launch at a distance step: counter held at 0
            state.zero_()
            L.sb200_mlp_forward_per_actor_f32(C.byref(dimg), stride, _p(x), D, N, _p(out), A, C.byref(d), _p(dist), 10,
                                              _p(state), st)
        ms_zero = events(lambda: state.zero_(), reps)
        ms_ad = events(adaptive, reps) - ms_zero
        wbytes = N * net.size * 4
        rows.append(dict(N=N, forward_us=ms_fwd * 1e3, forward_TBps=wbytes / (ms_fwd * 1e-3) / 1e12,
                         forward_share_of_3_35=wbytes / (ms_fwd * 1e-3) / 3.35e12, forward_floor_us=wbytes / 3.35e12 * 1e6,
                         forward_adaptive_us=ms_ad * 1e3, apply_us=ms_apply * 1e3,
                         apply_TBps=N * stride * 4 / (ms_apply * 1e-3) / 1e12))
        print(json.dumps(rows[-1]), flush=True)
        del images
    return rows


def acts(steps):
    from helpers import ddpg_configs
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.env import SyntheticEnv
    from surreal_b200.replay import UniformReplay
    from host_env_timing import HostEnv
    N = 1024
    out = []
    for kind in (None, 'normal', 'adaptive_normal'):
        for host in (True, False):
            lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=HID, critic_h=(400, 300), n_step=3, memory_size=200000, start=0)
            lc.algo.exploration.param_noise_type = kind
            ec.num_envs, ec.num_agents = N, N
            ec.limit_episode_length = steps
            UniformReplay(lc, ec, sc)
            ag = DDPGAgent(lc, ec, sc, 0, 'training')
            if kind is not None:
                ag.apply_param_noise()
            if host:
                env = HostEnv(N, D, A, steps, rew64=True)
                ag.env = w = ag.prepare_env_agent(env)
                obs, _ = w.reset()
                for _ in range(10):
                    ag.act(obs)
                torch.cuda.synchronize()
                t_act = 0.0
                for _ in range(steps):
                    t0 = time.perf_counter()
                    a = ag.act(obs)                    # ends in a stream synchronisation
                    t_act += time.perf_counter() - t0
                    obs, _, _, _ = w.step(a)
                torch.cuda.synchronize()
                ms = t_act / steps * 1e3
            else:
                ag.main_setup(SyntheticEnv(N, D, A, steps, seed=1))
                ag.main_loop(max_steps=steps)          # capture
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(3):
                    ag.main_loop(max_steps=steps)
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) / (3 * steps) * 1e3
            row = dict(param_noise=kind, path='host act()' if host else 'device chunk step (act + env + staging)',
                       N=N, ms=ms)
            print(json.dumps(row), flush=True)
            out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=200)
    ap.add_argument('--steps', type=int, default=64)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    import __graft_entry__
    __graft_entry__.build()
    res = dict(card=card(), kernels=kernels(a.reps), act=acts(a.steps))
    print(json.dumps(res['card']))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as fp:
            json.dump(res, fp, indent=1)


if __name__ == '__main__':
    main()

#!/usr/bin/env python
"""clock64 timeline of the persistent rollout kernel: builds a -DRF_TRACE variant of the library under tools/_trace/
(never the shipped .so), runs one chunk at the bench shape and prints how many clusters the device holds at once, in
how many waves the chunk's CTAs ran (every CTA's SM and %globaltimer at entry and exit), and, per phase, the cycles
cluster 0's CTAs spent.

    python tools/rollout_trace.py build      # nvcc only, no GPU needed
    python tools/rollout_trace.py            # one chunk of the agent alone
    python tools/rollout_trace.py engine     # every rollout of a few PipelinedEngine steps (learner running beside it)
"""
import ctypes as C
import glob
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
OUT = os.path.join(ROOT, 'tools', '_trace')
LIB = os.path.join(OUT, 'libsurreal_b200_trace.so')
# one-group stamps of thread 0 in step order after the step top (stamp 0), each timing the interval since the one before
NAMES = [(18, 'input-tile wait'), (3, 'L1 fma + push'), (4, 'H1 wait'), (7, 'L2 fma + push'), (9, 'H2 wait + head'),
         (10, 'head sync'), (11, 'phase 2 (sample+env)'), (12, 'commit_actor'), (13, 'x0 push')]


def build():
    from surreal_b200 import build as B
    os.makedirs(OUT, exist_ok=True)
    procs = []
    for src in B._sources():
        obj = os.path.join(OUT, os.path.basename(src)[:-3] + '.o')
        procs.append((obj, subprocess.Popen([B.NVCC] + B.FLAGS + ['-DRF_TRACE', '-c', src, '-o', obj], stdout=subprocess.PIPE,
                                            stderr=subprocess.STDOUT, text=True)))
    objs = []
    for obj, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            sys.stderr.write(out)
            raise SystemExit(1)
        objs.append(obj)
    subprocess.check_call([B.NVCC, '-shared', '-o', LIB] + objs + ['-lcudart'])
    print(LIB)


def waves(L, np):
    """Residency of the last chunk's launch: how many 4-CTA clusters the device can hold at once at this launch
    configuration, and in how many waves the CTAs actually ran (a CTA that starts after another has exited belongs
    to a later wave)."""
    cta = np.zeros((4096, 3), dtype=np.int64)
    info = np.zeros(4, dtype=np.int64)
    L.sb200_debug_rf_ctas.argtypes = [C.c_void_p, C.c_void_p]
    assert L.sb200_debug_rf_ctas(cta.ctypes.data_as(C.c_void_p), info.ctypes.data_as(C.c_void_p)) == 0
    grid, smem, groups, max_clusters = (int(v) for v in info)
    cta = cta[:grid]
    print('launch: %d CTAs = %d clusters of 4 (%d group(s) of 32 actors each), 512 threads, %d B dynamic shared memory; '
          'cudaOccupancyMaxActiveClusters = %d' % (grid, grid // 4, groups, smem, max_clusters))
    t0 = cta[:, 1].min()
    start, end = cta[:, 1] - t0, cta[:, 2] - t0
    wave = np.zeros(grid, dtype=np.int64)
    order = np.argsort(start, kind='stable')
    first_end = None
    w = 0
    for i in order:                                   # a new wave begins at the first CTA that starts after an exit
        if first_end is not None and start[i] >= first_end:
            w += 1
            first_end = None
        wave[i] = w
        first_end = end[i] if first_end is None else min(first_end, end[i])
    print('%d distinct SMs; %d wave(s); kernel span %.3f ms' % (len(set(cta[:, 0].tolist())), w + 1, end.max() / 1e6))
    for k in range(w + 1):
        sel = wave == k
        print('   wave %d: %3d CTAs, start %.3f..%.3f ms, end %.3f..%.3f ms, duration %.3f ms'
              % (k, sel.sum(), start[sel].min() / 1e6, start[sel].max() / 1e6, end[sel].min() / 1e6, end[sel].max() / 1e6,
                 (end[sel].max() - start[sel].min()) / 1e6))
    return groups


def two_groups(tr, np):
    """Cycle stamps of the two-group schedule, relative to the layer warps' step top (group 0's layer 1 begins)."""
    marks = [(3, 'layer warps: g0 layer 1 + H1 wait'), (4, 'layer warps: g0 layer 2'), (5, 'layer warps: g1 x0 wait + layer 1 + H1 wait'),
             (6, 'layer warps: g1 layer 2'), (8, 'tail warps: g0 tail starts'), (9, 'tail warps: g0 precompute + H2 wait'),
             (10, 'tail warps: g0 head'), (11, 'tail warps: g0 sample+env+commit'), (12, 'tail warps: g1 tail starts'),
             (13, 'tail warps: g1 precompute + H2 wait'), (14, 'tail warps: g1 head'), (15, 'tail warps: g1 sample+env+commit')]
    for cta in range(4):
        d = tr[cta]
        step = np.median(d[1:, 0] - d[:-1, 0])
        print('CTA %d: step period %.0f cycles (cycles since step top)' % (cta, step))
        for i, name in marks:
            print('   %-46s %7.0f' % (name, np.median(d[:, i] - d[:, 0])))


def main():
    import numpy as np
    import torch
    from surreal_b200 import _lib
    _lib.LIB_PATH = LIB
    from helpers import ppo_configs
    from surreal_b200.agent import PPOAgent
    from surreal_b200.replay import FIFOReplay
    from surreal_b200.env import SyntheticEnv
    N, D, A, T = 1024, 64, 8, 128
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=(256, 256), critic_h=(256, 256), n_step=128, stride=128, B=N, memory_size=4 * N)
    ec.num_envs = N
    R = FIFOReplay(lc, ec, sc)  # noqa: F841
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    env = SyntheticEnv(N, D, A, limit_episode_length=256, seed=0)
    ag.env = w = ag.prepare_env_agent(env)
    w.reset()
    for _ in range(3):
        ag.rollout_chunk(T)
    torch.cuda.synchronize()
    tr = np.zeros((4, 8, 32), dtype=np.int64)
    L = _lib.lib()
    groups = waves(L, np)
    L.sb200_debug_rf_trace.argtypes = [C.c_void_p]
    assert L.sb200_debug_rf_trace(tr.ctypes.data_as(C.c_void_p)) == 0
    if groups == 2:
        two_groups(tr, np)
        return
    for cta in range(4):
        print('CTA %d (cycles since step top; delta)' % cta)
        d = tr[cta]
        prev, total = 0, 0.0
        for i, name in NAMES:
            per = np.median(d[:, i] - d[:, prev])
            print('   %-24s %7.0f' % (name, per))
            prev, total = i, total + per
        step = np.median(d[1:, 0] - d[:-1, 0])
        print('   %-24s %7.0f   (step period %0.f)' % ('sum', total, step))
        print('   env warp: start %+.0f relative to step top, busy %0.f' % (np.median(d[:, 16] - d[:, 0]), np.median(d[:, 17] - d[:, 16])))
        print('   phase 2: slice sums %0.f | mean/sample/stores %0.f | env finalize %0.f | bookkeeping %0.f'
              % (np.median(d[:, 19] - d[:, 10]), np.median(d[:, 20] - d[:, 19]), np.median(d[:, 21] - d[:, 20]), np.median(d[:, 11] - d[:, 21])))


def engine(steps=8):
    """Waves of the rollout launched by each PipelinedEngine step at the bench shape: with the learner overlapped, its CTAs
    are resident next to the rollout's, and every step's rollout must still run in one wave."""
    import numpy as np
    import torch
    from surreal_b200 import _lib
    _lib.LIB_PATH = LIB
    import bench
    from surreal_b200.launch import SurrealDefaultLauncher, PipelinedEngine
    from surreal_b200.agent import PPOAgent
    from surreal_b200.learner import PPOLearner
    from surreal_b200.replay import FIFOReplay
    lc, ec, sc = bench.build_configs(bench.N_ACTORS, bench.HORIZON)
    agent, replay, learner = SurrealDefaultLauncher(PPOAgent, PPOLearner, FIFOReplay, sc, ec, lc).setup_engine()
    eng = PipelinedEngine(agent, replay, learner, bench.HORIZON)
    print('overlap: %s; learner SM budget %d (0: all SMs)' % (eng.overlap, learner.sm_budget))
    eng.prime()
    for _ in range(3):
        eng.step()
    torch.cuda.synchronize()
    L = _lib.lib()
    for k in range(steps):
        eng.step()
        print('step %d:' % k)
        waves(L, np)                                  # the rollout this step launched (synchronises the device)


if __name__ == '__main__':
    if len(sys.argv) > 1 and sys.argv[1] == 'build':
        build()
    elif len(sys.argv) > 1 and sys.argv[1] == 'engine':
        engine()
    else:
        main()

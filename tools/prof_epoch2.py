#!/usr/bin/env python
"""Phase profile of the one-launch learner kernel (csrc/epoch2.cu) at the bench shape: accumulated clock64 cycles per phase
(CTA 0 and the last CTA) over a few learn() calls, printed as microseconds per learn().

    python tools/prof_epoch2.py [clip|adapt] [--sm-budget N]    # N CTAs, as PipelinedEngine caps the learner (0: all SMs)
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def main():
    import numpy as np
    import torch
    from helpers import ppo_configs
    from surreal_b200.learner import PPOLearner
    B, n, D, A = 1024, 128, 64, 8
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument('mode', nargs='?', default='clip', choices=('clip', 'adapt'))
    ap.add_argument('--sm-budget', type=int, default=0)
    args = ap.parse_args()
    mode = args.mode
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=(256, 256), critic_h=(256, 256), n_step=n, stride=n, B=B, mode=mode, lr=1e-4)
    lc.algo.consts.kl_target = 1e6                      # no KL early stop: every policy epoch runs, as in the bench
    L = PPOLearner(lc, ec, sc)
    L.set_sm_budget(args.sm_budget)
    rng = np.random.default_rng(0)

    def batch():
        mean = np.tanh(rng.standard_normal((B, n, A)) * 0.3).astype(np.float32)
        std = np.exp(rng.uniform(-1.2, -0.6, (B, n, A))).astype(np.float32)
        return {'obs': (rng.standard_normal((B, n, D)) * 1.2).astype(np.float32),
                'obs_next': (rng.standard_normal((B, 1, D)) * 1.2).astype(np.float32),
                'actions': np.clip(rng.standard_normal((B, n, A)) * std + mean, -1, 1).astype(np.float32),
                'rewards': (rng.standard_normal((B, n)) * 0.3).astype(np.float32), 'dones': np.zeros((B, n), dtype=np.float32),
                'persistent_infos': [np.concatenate([mean, std], axis=2)], 'onetime_infos': None}
    b = batch()
    for _ in range(3):
        L.learn(b)
    torch.cuda.synchronize()
    pair = L._ek[3]
    assert pair is not None
    pair.profile(reset=True)
    pair.cta_profile()
    reps = 10
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    print('policy epochs of the last learn():', L.last_n_policy_epochs, '| SM budget:', args.sm_budget or 'all SMs')
    ev0.record()
    for _ in range(reps):
        pair.run()                                      # the kernel alone, on the resident batch
    ev1.record()
    torch.cuda.synchronize()
    print('sb200_ppo_epochs2_f32: %.1f us per launch' % (ev0.elapsed_time(ev1) / reps * 1e3))
    mhz = 1965.0
    tot0 = tot1 = 0.0
    for name, c0, c1 in pair.profile():
        u0, u1 = c0 / reps / mhz, c1 / reps / mhz
        tot0 += u0
        tot1 += u1
        print('  %-12s CTA 0 %8.1f us   last CTA %8.1f us' % (name, u0, u1))
    print('  %-12s CTA 0 %8.1f us   last CTA %8.1f us' % ('sum', tot0, tot1))
    cp = pair.cta_profile()
    print('per-CTA us per launch: P1 | P2 | forward (GEMMs) | loss rows + d2 | d1 GEMM')
    for c in list(range(0, 132, 8)) + [60, 61, 62, 63, 123, 124, 125, 126, 127]:
        v = [x / reps / mhz for x in cp[c]]
        print('  CTA %3d: %7.1f | %7.1f | %7.1f (%7.1f) | %7.1f | %7.1f' % (c, v[0], v[1], v[2], v[3], v[4], v[5]))


if __name__ == '__main__':
    main()

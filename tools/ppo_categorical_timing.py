#!/usr/bin/env python
"""Timing of the categorical PPO policy (csrc/ppo_cat.cu), one process, CUDA events after warm-up:

  act     PPOAgent.act() per step at 1024 actors on the device-resident discrete synthetic env (64-dim observations,
          2x256 MLP policy, the per-step launch chain), K = 4 and K = 18, against the Gaussian policy with A = 8;
  learn   learn() at BASELINE configs[1]'s shape (batch 1024 x n_step 128, 64-dim observations, 2x256 actor and critic,
          captured graph), the categorical policy with K = 18 against the Gaussian policy with A = 8, both on the
          launch chain (the one-launch epoch kernel is Gaussian only).  Arms alternate within each round.
The card's name, power limit and maximum SM clock are read in the same run.

    python tools/ppo_categorical_timing.py [--rounds 3] [--out ppo_categorical_timing.json]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

D, N, H = 64, 1024, 256


def configs(K, discrete, B=1024, n=128):
    from surreal_b200.session import Config
    from surreal_b200.main.ppo_configs import (PPO_DEFAULT_LEARNER_CONFIG, PPO_DEFAULT_ENV_CONFIG,
                                               PPO_DEFAULT_SESSION_CONFIG)
    lc = Config(copy.deepcopy(PPO_DEFAULT_LEARNER_CONFIG.to_dict()))
    ec = Config(copy.deepcopy(PPO_DEFAULT_ENV_CONFIG.to_dict()))
    sc = Config(copy.deepcopy(PPO_DEFAULT_SESSION_CONFIG.to_dict()))
    sc.folder = tempfile.mkdtemp()
    ec.env_name, ec.num_envs, ec.num_agents, ec.limit_episode_length = 'synthetic', N, N, 200
    ec.obs_spec = {'low_dim': {'flat_inputs': (D,)}}
    ec.action_spec = {'dim': (K,), 'type': 'discrete' if discrete else 'continuous'}
    lc.model.actor_fc_hidden_sizes = lc.model.critic_fc_hidden_sizes = [H, H]
    lc.algo.ppo_mode = 'clip'
    lc.algo.rnn.if_rnn_policy = False
    lc.algo.n_step = lc.algo.stride = n
    lc.replay.batch_size = B
    lc.replay.memory_size = 4 * N
    lc.parameter_publish.exp_interval = B
    return lc, ec, sc


def events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def act_arm(K, discrete):
    from surreal_b200.agent import PPOAgent
    from surreal_b200.replay import FIFOReplay
    lc, ec, sc = configs(K, discrete)
    FIFOReplay(lc, ec, sc)
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    ag.env = w = ag.prepare_env_agent(ag.get_env())
    state = {'obs': w.reset()[0]}

    def step():
        a = ag.act(state['obs'])
        state['obs'] = w.step(a)[0]
    return step


def learn_arm(K, discrete):
    from surreal_b200.learner import PPOLearner
    lc, ec, sc = configs(K, discrete)
    L = PPOLearner(lc, ec, sc)
    L.use_epoch_kernel = False                      # the launch chain for both policies
    L.tensorplex.add_scalars = lambda *a, **k: None
    L.periodic_checkpoint = lambda *a, **k: None
    B, n = 1024, 128
    rng = np.random.default_rng(K)
    obs = (rng.standard_normal((B, n, D)) * 1.2).astype(np.float32)
    if discrete:
        lg = rng.standard_normal((B * n, K))
        p = np.exp(lg - lg.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        pd = np.concatenate([p, np.log(p)], 1).astype(np.float32).reshape(B, n, 2 * K)
        actions = np.eye(K, dtype=np.float32)[rng.integers(0, K, (B, n))]
    else:
        pd = np.concatenate([rng.uniform(-0.5, 0.5, (B, n, K)), np.full((B, n, K), np.exp(-1.0))], 2).astype(np.float32)
        actions = np.clip(rng.standard_normal((B, n, K)) * 0.37, -1, 1).astype(np.float32)
    dev = lambda x: torch.tensor(x, device='cuda')  # noqa: E731
    batch = {'obs': {'low_dim': {'flat_inputs': dev(obs)}}, 'obs_next': {'low_dim': {'flat_inputs': dev(obs[:, :1])}},
             'actions': dev(actions), 'rewards': dev((rng.standard_normal((B, n)) * 0.3).astype(np.float32)),
             'dones': dev(np.zeros((B, n), np.float32)), 'persistent_infos': [dev(pd)], 'onetime_infos': None}
    return lambda: L.learn(batch)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--act-steps', type=int, default=400)
    ap.add_argument('--learn-iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('ppo_categorical_timing needs a CUDA device')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    res = {'card': torch.cuda.get_device_name(0), 'nvidia_smi': smi}
    acts = {'cat_K4': act_arm(4, True), 'cat_K18': act_arm(18, True), 'gauss_A8': act_arm(8, False)}
    learns = {'cat_K18': learn_arm(18, True), 'gauss_A8': learn_arm(8, False)}
    for fn in list(acts.values()):
        events_ms(fn, 50)                            # warm-up
    for fn in list(learns.values()):
        events_ms(fn, 3)
    t_act = {k: [] for k in acts}
    t_learn = {k: [] for k in learns}
    for _ in range(args.rounds):
        for k, fn in acts.items():
            t_act[k].append(events_ms(fn, args.act_steps))
        for k, fn in learns.items():
            t_learn[k].append(events_ms(fn, args.learn_iters))
    med = lambda v: {'median_ms': float(np.median(v)), 'min_ms': float(np.min(v)), 'max_ms': float(np.max(v))}  # noqa: E731
    res['act_step_1024_actors'] = {k: med(v) for k, v in t_act.items()}
    res['learn_1024x128'] = {k: med(v) for k, v in t_learn.items()}
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as fp:
            json.dump(res, fp, indent=1)


if __name__ == '__main__':
    main()

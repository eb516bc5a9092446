#!/usr/bin/env python
"""Generate the golden vectors of n-step SSAR staging for several actors by running the REAL reference, with the harness
and helpers of make_golden.py (run in the build container only, like it):

    python tests/golden/make_golden_ssar_multi.py          # writes window_ssar_multi.npz

  fixture                  reference code that produced it
  -----------------------  ----------------------------------------------------------------------------------------------
  window_ssar_multi.npz    ExpSenderWrapperSSARNStepBootstrap._reset / _step (exp_sender_wrapper.py:72-112), one wrapper
                           per actor, all sending into one sink in (step, actor) order

Every (n_step, gamma) of {1, 2, 3, 5} x {0, 1, 0.37, 0.99}: 5 actors over 30 steps, each actor with its own episode
script (length-1 episodes, episodes shorter than n_step, episodes ending on an emission step, staggered ends).  Rewards
are float64 N(0, 3) draws with full 53-bit mantissas.  Observations encode (actor, step): the successor of actor a after
its g-th step is 1000 a + g, the observation reset() returns is 1000 a + g + 0.5, the action is 1000 a + g + 0.25.
Stored per case: every sent record in send order (and the step that sent it), and after every step each actor's pending
deque -- length, obs, action, and the running reward sums as float64 bits.  The file is written with fixed zip
timestamps, so a re-run gives the same bytes."""
import json
import os
import sys
import zipfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (installs the reference harness)

import numpy as np  # noqa: E402

ESW = G.ESW
OUT = os.path.join(G.HERE, 'window_ssar_multi.npz')
N_ACT, T = 5, 30


class _Actor:
    """One actor's env: scripted episode lengths (cycled), rewards from a fixed float64 array."""
    metadata = {}

    def __init__(self, a, script, rewards):
        self.a, self.script, self.rew = a, script, rewards
        self.g = self.t = self.ep = 0

    def reset(self):
        self.t = 0
        return 1000.0 * self.a + self.g + 0.5, {}

    def step(self, action):
        self.g += 1
        self.t += 1
        done = self.t >= self.script[self.ep % len(self.script)]
        if done:
            self.ep += 1
        return 1000.0 * self.a + self.g, float(self.rew[self.g - 1]), done, {}

    def close(self):
        pass


def _scripts(n):
    return [[1, 1, 4, 1],                       # length-1 episodes
            [n, n, 2 * n + 1],                  # ends exactly on an emission step
            [max(n - 1, 1), 7, 2],              # shorter than n_step (never emits for n > 1)
            [T + 5],                            # never ends within the run
            [3, 5, 2, 6]]                       # staggered


def run_case(n, gamma, seed):
    lc, ec, sc = G.cfg_ddpg(n_step=n)
    lc.algo.gamma = gamma
    rng = np.random.default_rng(seed)
    rew = rng.standard_normal((N_ACT, T)) * 3.0
    scripts = _scripts(n)
    sink = G._Sink()
    envs = [_Actor(a, scripts[a], rew[a]) for a in range(N_ACT)]
    ws = []
    for e in envs:
        w = ESW.ExpSenderWrapperSSARNStepBootstrap(e, lc, sc)
        w.sender = sink
        ws.append(w)
    obs0 = np.array([w.reset()[0] for w in ws])
    obs_next = np.zeros((T, N_ACT))
    obs_reset = np.zeros((T, N_ACT))
    action = np.zeros((T, N_ACT))
    done = np.zeros((T, N_ACT), np.uint8)
    pend_len = np.zeros((T, N_ACT), np.int32)
    pend_obs = np.zeros((T, N_ACT, n))
    pend_act = np.zeros((T, N_ACT, n))
    pend_sum = np.zeros((T, N_ACT, n), np.uint64)
    rec_step = []
    for t in range(T):
        for a, (w, e) in enumerate(zip(ws, envs)):
            action[t, a] = 1000.0 * a + e.g + 0.25
            before = len(sink.sent)
            on, r, d, _ = w.step(action[t, a])
            rec_step += [t] * (len(sink.sent) - before)
            obs_next[t, a], done[t, a] = on, d
            obs_reset[t, a] = w.reset()[0] if d else on
        for a, w in enumerate(ws):
            pend_len[t, a] = len(w.last_n)
            for k, ex in enumerate(w.last_n):
                pend_obs[t, a, k], pend_act[t, a, k] = ex[0][0], ex[1]
                pend_sum[t, a, k] = np.array(ex[2], np.float64).view(np.uint64)
    rec = dict(obs=[h['obs'][0] for h, _ in sink.sent], obs_next=[h['obs'][1] for h, _ in sink.sent],
               act=[x['action'] for _, x in sink.sent], rew=[x['reward'] for _, x in sink.sent],
               done=[x['done'] for _, x in sink.sent])
    arrs = dict(rew=rew.T.copy(), obs0=obs0, obs_next=obs_next, obs_reset=obs_reset, action=action, done=done,
                pend_len=pend_len, pend_obs=pend_obs, pend_act=pend_act, pend_sum=pend_sum,
                rec_step=np.array(rec_step, np.int32),
                rec_obs=np.array(rec['obs'], np.float64), rec_obs_next=np.array(rec['obs_next'], np.float64),
                rec_act=np.array(rec['act'], np.float64), rec_rew=np.array(rec['rew'], np.float64),
                rec_done=np.array(rec['done'], np.uint8))
    return dict(n_step=n, gamma=gamma, N=N_ACT, T=T, scripts=scripts), arrs


def save_fixed(path, arrs):
    """np.savez_compressed with a fixed timestamp on every member."""
    with zipfile.ZipFile(path, 'w', compression=zipfile.ZIP_DEFLATED) as z:
        for k, v in arrs.items():
            zi = zipfile.ZipInfo(k + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            with z.open(zi, 'w', force_zip64=True) as fp:
                np.lib.format.write_array(fp, np.asanyarray(v), allow_pickle=False)
    print('wrote %-28s %7.1f KB' % (os.path.basename(path), os.path.getsize(path) / 1024))


def main():
    cases, out = [], {}
    k = 0
    for n in (1, 2, 3, 5):
        for gamma in (0.0, 1.0, 0.37, 0.99):
            meta, arrs = run_case(n, gamma, seed=100 + k)
            cases.append(meta)
            out.update({'c%d/%s' % (k, name): v for name, v in arrs.items()})
            k += 1
    out['cases'] = np.array(json.dumps(cases))
    save_fixed(OUT, out)


if __name__ == '__main__':
    main()

#!/usr/bin/env python
"""Generate the DQN golden vectors by RUNNING the real reference code through tests/golden/_ref_harness.py:

    python tests/golden/make_golden_dqn.py

  fixture                      reference code that produced it
  ---------------------------  ------------------------------------------------------------------------------------
  dqn_optimize_{tag}.npz       DQNLearner.learn / _optimize / _update_target (learner/dqn.py:10-92) with the Q function
                               of build_ffqfunc / DuelingQbase.forward (model/q_net.py:9-65,122-134), tag in
                               {duel, noduel} x {double, single}: six updates (the first through learn(), i.e. unit
                               weights; the rest through _optimize with non-unit importance weights followed by learn's
                               own tracker step, as the commented prioritized train_batch does, dqn.py:128-175), batch 16,
                               target period 40 samples (not a multiple of the batch: the third and fifth updates copy)
  dqn_qnet.npz                 DuelingQbase.forward on injected weights, dueling on and off
  dqn_explore.npz              QAgent.act (agent/q_agent.py:35-53) in training mode for both schedules, with the
                               random.random() / random.randrange() draws it consumed recorded
  dqn_reference.npz            LinearSchedule / PiecewiseSchedule.value (utils/schedule.py:34-99) over a grid of t, and the
                               literal default_config trees of DQNLearner and QAgent (dqn.py:94-121, q_agent.py:55-65)

dqn.py cannot run as shipped: it calls U.huber_loss_per_element, U.conv_fc_init, U.infer_shape_conv2d and torchx's
Module.clone / copy_from / clip_grad_norm, none of which exists in the reference.  They are registered HERE, as
DESIGN.md §4 decides them (openai-baselines Huber with delta 1, a deep copy, a parameter copy,
torch.nn.utils.clip_grad_norm_); the harness is left as it is.  Weights are injected.

Every case has terminal rows, TD errors on both sides of the Huber kink, and exact ties: the action tower's last layer
has identical rows (and biases) 1 and 3, and the batches never take actions 1 or 3, so those two Q columns receive
identical gradients and stay exactly equal through every update (a double-Q argmax at s' that lands on them must take
column 1, the first index).  Away from those ties every argmax / max at s' has a top-2 margin of at least MARGIN, checked
here, so that its choice cannot depend on the rounding order of another implementation.
"""
import ast
import copy
import importlib.util
import json
import os
import random
import sys
import warnings
import tempfile

import numpy as np
import torch

warnings.filterwarnings('ignore')
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _ref_harness as H  # noqa: E402

H.install()
import surreal.utils as U  # noqa: E402
import torch.nn as nn  # noqa: E402

REF = H.REF_ROOT + '/surreal'
B, D, NA, HID, PERIOD, GAMMA, LR, ITERS = 16, 8, 5, [12, 10], 40, 0.99, 1e-3, 6
TIE = (1, 3)
MARGIN = 1e-3
T_GRID = np.array([0, 1, 7, 99, 100, 101, 250, 999, 1000, 1001, 5000, 10 ** 6], dtype=np.int64)


# ---- the stand-ins the reference's DQN needs and does not ship (DESIGN.md §4) ---------------------------------------
def huber_loss_per_element(x, delta=1.0):
    """openai-baselines huber_loss: 0.5 x^2 for |x| < delta, delta (|x| - 0.5 delta) otherwise."""
    return torch.where(x.abs() < delta, 0.5 * x * x, delta * (x.abs() - 0.5 * delta))


U.huber_loss_per_element = huber_loss_per_element
U.conv_fc_init = lambda layer: None                      # weights are injected below
U.infer_shape_conv2d = lambda *a, **k: (_ for _ in ()).throw(NotImplementedError('convs'))
U.is_valid_shape = lambda shape: all(int(s) > 0 for s in shape)
U.flatten_conv = lambda x: x.view(x.size(0), -1)
U.shape = lambda t: tuple(t.size())
U.to_scalar = lambda t: float(t.item()) if hasattr(t, 'item') else float(t)
U.torch_ones_like = torch.ones_like
TxModule = sys.modules['torchx.nn'].Module
TxModule.clone = lambda self: copy.deepcopy(self)
TxModule.copy_from = lambda self, other: self.load_state_dict(other.state_dict())
TxModule.clip_grad_norm = lambda self, max_norm: nn.utils.clip_grad_norm_(self.parameters(), max_norm)

from surreal.session import Config  # noqa: E402
from surreal.main.ddpg_configs import DDPG_DEFAULT_SESSION_CONFIG  # noqa: E402
from surreal.learner.dqn import DQNLearner  # noqa: E402
import surreal.agent.q_agent as q_agent_mod  # noqa: E402


def save(name, **arrs):
    out = {}
    for k, v in arrs.items():
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu().numpy()
        if isinstance(v, (dict, list, str)) and not isinstance(v, np.ndarray):
            v = np.array(json.dumps(v))
        out[k] = np.asarray(v)
    path = os.path.join(HERE, name + '.npz')
    np.savez_compressed(path, **out)
    print('wrote %-26s %7.1f KB' % (name + '.npz', os.path.getsize(path) / 1024))


def sd_np(module, prefix=''):
    return {prefix + k.replace('.', '/'): v.detach().cpu().numpy().copy() for k, v in module.state_dict().items()}


def configs(dueling, double_q):
    lc = Config({'model': {'convs': [], 'fc_hidden_sizes': list(HID), 'dueling': dueling},
                 'algo': {'lr': LR, 'optimizer': 'Adam', 'grad_norm_clipping': 10, 'gamma': GAMMA,
                          'target_network_update_freq': PERIOD, 'double_q': double_q,
                          'exploration': {'schedule': 'linear', 'steps': 1000, 'final_eps': 0.02}},
                 'eval': {'eps': 0.05}, 'replay': {'batch_size': B}})
    ec = Config({'obs_spec': {'dim': (D,)}, 'action_spec': {'dim': (NA,), 'type': 'discrete'}})
    sc = Config(copy.deepcopy(DDPG_DEFAULT_SESSION_CONFIG.to_dict()))   # the plumbing trees the base classes read
    sc.folder = tempfile.mkdtemp()
    return lc, ec, sc


def inject(q_func, g):
    """Seeded weights; rows TIE of the action tower's last layer (and their biases) equal."""
    with torch.no_grad():
        for p in q_func.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (0.5 if p.dim() == 2 else 0.2))
        last = q_func.fc_action_layers[-1]
        last.weight[TIE[1]].copy_(last.weight[TIE[0]])
        last.bias[TIE[1]].copy_(last.bias[TIE[0]])


def margin_ok(q):
    """Every row's largest value is at least MARGIN above its next distinct value (exactly equal columns count once)."""
    for row in q:
        u = torch.unique(row)
        if u.numel() > 1 and float(u[-1] - u[-2]) < MARGIN:
            return False
    return True


def gen_optimize(dueling, double_q):
    tag = ('duel' if dueling else 'noduel') + '_' + ('double' if double_q else 'single')
    lc, ec, sc = configs(dueling, double_q)
    L = H.construct_without_initialize(DQNLearner, lc, ec, sc)
    L.tensorplex = H._Any()
    g = torch.Generator().manual_seed(31 + 2 * dueling + double_q)
    inject(L.q_func, g)
    L.q_target.copy_from(L.q_func)
    with torch.no_grad():                                # target != online at the start: the target path is exercised
        for p in L.q_target.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=g))
        last = L.q_target.fc_action_layers[-1]           # the target's tied columns DIFFER: the tie rule matters
        last.bias[TIE[1]].add_(0.5)
    out = dict(**sd_np(L.q_func, 'init/model/'), **sd_np(L.q_target, 'init/target/'))
    rng = np.random.default_rng(41 + 2 * dueling + double_q)
    tds, stats = [], []
    it = 0
    while it < ITERS:
        raw = dict(obs=rng.standard_normal((B, D)).astype(np.float32),
                   obs_next=rng.standard_normal((B, D)).astype(np.float32),
                   actions=rng.choice([0, 2, 4], size=(B, 1)).astype(np.int64),
                   rewards=(rng.standard_normal((B, 1)) * 1.5).astype(np.float32),
                   dones=(rng.random((B, 1)) < 0.25).astype(np.float32),
                   weights=(rng.uniform(0.3, 1.7, (B, 1)) if it > 0 else np.ones((B, 1))).astype(np.float32))
        raw['dones'][0] = 1.0                            # at least one terminal row per batch
        t = {k: torch.from_numpy(v) for k, v in raw.items()}
        with torch.no_grad():
            q_on, q_tg = L.q_func(t['obs_next']), L.q_target(t['obs_next'])
        if not (margin_ok(q_on) and margin_ok(q_tg)):
            continue                                     # redraw this batch (the generator state moves on)
        on_arg = q_on.max(1)[1]
        if double_q and not bool((on_arg == TIE[0]).any()):
            continue                                     # every double-Q case takes the tie branch at least once
        assert bool((q_on[:, TIE[0]] == q_on[:, TIE[1]]).all())
        if it == 0:
            batch = H._AttrDict(obs=t['obs'], actions=t['actions'], rewards=t['rewards'], obs_next=t['obs_next'],
                                dones=t['dones'])
            captured = {}
            orig = L._optimize

            def spy(*a):
                captured['td'] = orig(*a)
                return captured['td']
            L._optimize = spy
            L.learn(batch)                                # unit weights + learn()'s own target tracker
            del L._optimize
            td = captured['td']
        else:
            td = L._optimize(t['obs'], t['actions'], t['rewards'], t['obs_next'], t['dones'], t['weights'])
            if L.target_update_tracker.track_increment(B):                  # dqn.py:84-86
                L._update_target()
        td = td.detach().view(-1)
        a = td.abs()
        assert bool((a < 1).any()) and bool((a > 1).any()), 'both Huber branches in every batch'
        w = t['weights'].view(-1).double()
        stats.append({'td_error': float(a.double().mean()),
                      'loss': float((w * huber_loss_per_element(td.double())).mean()),
                      'tie_rows': int((on_arg == TIE[0]).sum())})
        tds.append(td.numpy().copy())
        for k, v in raw.items():
            out['it%d/%s' % (it, k)] = v
        out.update(sd_np(L.q_func, 'it%d/model/' % it))
        out.update(sd_np(L.q_target, 'it%d/target/' % it))
        it += 1
    lw = L.q_func.fc_action_layers[-1]
    assert torch.equal(lw.weight[TIE[0]], lw.weight[TIE[1]]) and torch.equal(lw.bias[TIE[0]], lw.bias[TIE[1]])
    cfg = dict(B=B, D=D, n_actions=NA, hidden=HID, dueling=dueling, double_q=double_q, gamma=GAMMA, lr=LR,
               period=PERIOD, grad_norm_clipping=10, tie=list(TIE), iters=ITERS,
               target_copies=[i for i in range(ITERS) if (i + 1) * B // PERIOD > i * B // PERIOD])
    save('dqn_optimize_' + tag, cfg=cfg, stats=stats, td=np.stack(tds), **out)


def gen_qnet():
    out = {}
    g = torch.Generator().manual_seed(7)
    x = torch.randn(33, D, generator=g)
    out['x'] = x.numpy()
    for dueling in (False, True):
        lc, ec, sc = configs(dueling, True)
        L = H.construct_without_initialize(DQNLearner, lc, ec, sc)
        inject(L.q_func, g)
        with torch.no_grad():
            q = L.q_func(x)
        tag = 'duel' if dueling else 'noduel'
        out.update(sd_np(L.q_func, tag + '/model/'))
        out[tag + '/q'] = q.numpy()
    save('dqn_qnet', **out)


class _Recorder:
    """Stands in for the module-level `random` of q_agent.py: the same seeded stream, every draw recorded."""

    def __init__(self, seed):
        self.r = random.Random(seed)
        self.log = []

    def random(self):
        u = self.r.random()
        self.log.append(('u', u))
        return u

    def randrange(self, n):
        a = self.r.randrange(n)
        self.log.append(('a', a))
        return a


def gen_explore():
    out = {}
    for sched, exp in (('linear', {'schedule': 'linear', 'steps': 40, 'final_eps': 0.1}),
                       ('piecewise', {'schedule': 'piecewise', 'steps': [10, 30], 'final_eps': [0.5, 0.05]})):
        lc, ec, sc = configs(True, True)
        lc.algo.exploration = Config(exp)
        Ag = H.construct_without_initialize(q_agent_mod.QAgent, lc, ec, sc, 0, 'training')
        g = torch.Generator().manual_seed(5)
        inject(Ag.q_func, g)
        rec = _Recorder(17)
        q_agent_mod.random = rec
        xs = torch.randn(60, D, generator=g)
        rows = []
        for T in range(60):
            eps = Ag.exploration.value(Ag.T)
            n0 = len(rec.log)
            with torch.no_grad():
                a = Ag.act(xs[T])
            draws = rec.log[n0:]
            u = draws[0][1]
            ra = draws[1][1] if len(draws) > 1 else -1
            rows.append((T, eps, u, ra, int(a)))
        q_agent_mod.random = random
        out.update(sd_np(Ag.q_func, sched + '/model/'))
        out[sched + '/x'] = xs.numpy()
        out[sched + '/rows'] = np.array(rows, dtype=np.float64)         # T, eps, u, random action (-1: none), action
        out[sched + '/exploration'] = np.array(json.dumps(exp))
    save('dqn_explore', **out)


def _schedule_module():
    spec = importlib.util.spec_from_file_location('schedule', os.path.join(REF, 'utils', 'schedule.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _default_config(path, cls):
    tree = ast.parse(open(path).read())
    for node in ast.walk(tree):
        if isinstance(node, ast.ClassDef) and node.name == cls:
            for fn in node.body:
                if isinstance(fn, ast.FunctionDef) and fn.name == 'default_config':
                    ret = next(s for s in fn.body if isinstance(s, ast.Return))
                    return ast.literal_eval(ret.value)
    raise KeyError(cls)


def gen_reference():
    S = _schedule_module()
    lin = S.LinearSchedule(schedule_timesteps=1000, final_p=0.02, initial_p=1.0)
    steps, finals = [100, 1000, 5000], [0.3, 0.05, 0.01]
    pw = S.PiecewiseSchedule(endpoints=[(0, 1.0)] + list(zip(steps, finals)), outside_value=finals[-1])
    np.savez(os.path.join(HERE, 'dqn_reference.npz'), t=T_GRID, linear=np.array([lin.value(int(t)) for t in T_GRID]),
             piecewise=np.array([pw.value(int(t)) for t in T_GRID]), piecewise_steps=np.array(steps),
             piecewise_final_eps=np.array(finals),
             learner_default_config=np.array(json.dumps(_default_config(os.path.join(REF, 'learner', 'dqn.py'),
                                                                        'DQNLearner'))),
             agent_default_config=np.array(json.dumps(_default_config(os.path.join(REF, 'agent', 'q_agent.py'),
                                                                      'QAgent'))))
    print('wrote dqn_reference.npz')


def main():
    torch.set_num_threads(1)
    for dueling in (True, False):
        for double_q in (True, False):
            gen_optimize(dueling, double_q)
    gen_qnet()
    gen_explore()
    gen_reference()


if __name__ == '__main__':
    main()

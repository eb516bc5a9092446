"""DQN on the CPU: the schedules and default config trees against the reference (tests/golden/dqn_reference.npz), the
float64 oracle's TD arithmetic, the configurations DQN rejects, the record layout of discrete specs and the act draws."""
import copy
import json

import numpy as np
import pytest
import torch

from oracle import dqn as odqn


def test_schedules_match_the_reference(golden):
    from surreal_b200 import utils as U
    from surreal_b200.agent.q_agent import exploration_schedule
    from surreal_b200.session import Config
    g = golden('dqn_reference')
    lin = exploration_schedule(Config({'schedule': 'linear', 'steps': 1000, 'final_eps': 0.02}))
    pw = exploration_schedule(Config({'schedule': 'piecewise', 'steps': [int(s) for s in g['piecewise_steps']],
                                      'final_eps': [float(e) for e in g['piecewise_final_eps']]}))
    for k, t in enumerate(g['t']):
        assert lin.value(int(t)) == g['linear'][k]
        assert pw.value(int(t)) == g['piecewise'][k]
    # the device form of the linear schedule: the same double arithmetic as the piecewise restatement
    P = U.LinearSchedule(1000, 0.02).device_points()
    pl = U.PiecewiseSchedule(list(zip(P[:2], P[2:4])), outside_value=P[4])
    assert all(pl.value(int(t)) == g['linear'][k] for k, t in enumerate(g['t']))


def test_default_configs_match_the_reference_trees(golden):
    from surreal_b200.main.dqn_configs import DQN_DEFAULT_LEARNER_CONFIG
    g = golden('dqn_reference')
    ref_l = json.loads(str(g['learner_default_config']))
    ref_a = json.loads(str(g['agent_default_config']))
    ours = DQN_DEFAULT_LEARNER_CONFIG.to_dict()
    assert ours['model'] == ref_l['model'] == ref_a['model']
    assert ours['eval'] == ref_a['eval']
    for k, v in ref_l['algo'].items():
        assert ours['algo'][k] == v, k
    assert ours['algo']['n_step'] == 1


def _configs(**over):
    from surreal_b200.session import Config
    from surreal_b200.main.dqn_configs import (DQN_DEFAULT_LEARNER_CONFIG, DQN_DEFAULT_ENV_CONFIG,
                                               make_discrete_synthetic_env_config)
    lc = Config(copy.deepcopy(DQN_DEFAULT_LEARNER_CONFIG.to_dict()))
    ec = Config(copy.deepcopy(DQN_DEFAULT_ENV_CONFIG.to_dict()))
    make_discrete_synthetic_env_config(ec, 4, 10, 5)
    lc.model.convs, lc.model.fc_hidden_sizes, lc.model.dueling = [], [16], True
    for k, v in over.items():
        if k == 'n_step':
            lc.algo.n_step = v
        elif k == 'convs':
            lc.model.convs = v
        elif k == 'continuous':
            ec.action_spec = {'dim': (5,), 'type': 'continuous'}
    return lc, ec


def test_rejections():
    from surreal_b200.learner.dqn import check_dqn_config
    from surreal_b200.session import ConfigError
    check_dqn_config(*_configs())
    with pytest.raises(ConfigError):
        check_dqn_config(*_configs(n_step=3))
    with pytest.raises(NotImplementedError):
        check_dqn_config(*_configs(convs=[[16, 8, 4]]))
    with pytest.raises(ConfigError):
        check_dqn_config(*_configs(continuous=True))


def test_record_layout_of_discrete_specs():
    from surreal_b200.utils import record_action_dim, action_is_discrete
    assert record_action_dim({'dim': (18,), 'type': 'discrete'}) == 1
    assert record_action_dim({'dim': (6,), 'type': 'continuous'}) == 6
    assert record_action_dim({'dim': (6,)}) == 6
    assert action_is_discrete({'dim': (2,), 'type': 'discrete'})


def test_aggregator_still_rejects_discrete_specs():
    from surreal_b200.learner import SSARAggregator
    with pytest.raises(Exception):
        SSARAggregator({'low_dim': {'flat_inputs': (4,)}}, {'dim': (3,), 'type': 'discrete'})


def test_oracle_huber_and_td_gradient():
    x = torch.tensor([-2.5, -1.0, -0.3, 0.0, 0.7, 1.0, 3.0], dtype=torch.float64, requires_grad=True)
    h = odqn.huber(x)
    assert torch.allclose(h, torch.tensor([2.0, 0.5, 0.045, 0.0, 0.245, 0.5, 2.5], dtype=torch.float64))
    h.sum().backward()
    assert torch.equal(x.grad, x.detach().clamp(-1, 1))
    # double Q picks the target column by the online argmax; a terminal row bootstraps nothing
    qa = torch.tensor([[1.0, 2.0, 0.0]], dtype=torch.float64)
    ta = torch.tensor([[5.0, -1.0, 9.0]], dtype=torch.float64)
    oa = torch.tensor([[0.0, 3.0, 1.0]], dtype=torch.float64)
    a, r = torch.tensor([1.0]), torch.tensor([0.5], dtype=torch.float64)
    _, td = odqn.td_loss(qa, None, ta, None, oa, None, a, r, torch.zeros(1), None, 0.9)
    assert float(td) == 2.0 - (0.5 + 0.9 * -1.0)
    _, td = odqn.td_loss(qa, None, ta, None, None, None, a, r, torch.zeros(1), None, 0.9)
    assert float(td) == 2.0 - (0.5 + 0.9 * 9.0)
    _, td = odqn.td_loss(qa, None, ta, None, None, None, a, r, torch.ones(1), None, 0.9)
    assert float(td) == 2.0 - 0.5


def test_act_draws_are_uniform_over_the_actions():
    u, a = odqn.act_draws(3, 7, np.arange(60000), 6)
    assert 0.0 <= u.min() and u.max() < 1.0
    counts = np.bincount(a, minlength=6)
    assert counts.min() > 9000 and counts.max() < 11000
    assert abs(u.mean() - 0.5) < 0.01


# ---- the oracle against goldens produced by running the reference's DQNLearner, DuelingQbase and QAgent ----------------
CASES = ['duel_double', 'duel_single', 'noduel_double', 'noduel_single']


def golden_layers(g, prefix, tower):
    """[(weight, bias)] of fc_{tower}_layers under ``prefix`` of a golden (None when the tower is absent)."""
    out, i = [], 0
    while '%sfc_%s_layers/%d/weight' % (prefix, tower, i) in g:
        p = '%sfc_%s_layers/%d/' % (prefix, tower, i)
        out.append((torch.from_numpy(g[p + 'weight']), torch.from_numpy(g[p + 'bias'])))
        i += 1
    return out or None


@pytest.mark.parametrize('case', CASES)
def test_oracle_learner_against_reference_goldens(golden, case):
    g = golden('dqn_optimize_' + case)
    cfg, stats = g.js('cfg'), g.js('stats')
    O = odqn.OracleDQN(golden_layers(g, 'init/model/', 'action'), golden_layers(g, 'init/model/', 'state'), cfg['lr'],
                       cfg['gamma'], cfg['double_q'], cfg['period'], cfg['grad_norm_clipping'],
                       target_action_layers=golden_layers(g, 'init/target/', 'action'),
                       target_state_layers=golden_layers(g, 'init/target/', 'state'))
    for it in range(cfg['iters']):
        p = 'it%d/' % it
        w = g[p + 'weights'] if it > 0 else None
        so = O.update(g[p + 'obs'], g[p + 'actions'], g[p + 'rewards'], g[p + 'obs_next'], g[p + 'dones'], w)
        assert np.abs(so['td'].numpy() - g['td'][it]).max() <= 1e-5, it
        for k in ('td_error', 'loss'):
            assert abs(so[k] - stats[it][k]) <= 1e-6 * max(1.0, abs(stats[it][k])), (it, k)
        for net, tgt in (('model', False), ('target', True)):
            for tower in ('action', 'state'):
                ref = golden_layers(g, p + net + '/', tower)
                if ref is None:
                    continue
                mine = (O.ta if tower == 'action' else O.tv) if tgt else (O.a if tower == 'action' else O.v)
                for (w_, b_), (rw, rb) in zip(mine, ref):
                    assert torch.allclose(w_.detach(), rw.double(), atol=1e-6), (it, net, tower)
                    assert torch.allclose(b_.detach(), rb.double(), atol=1e-6), (it, net, tower)
    assert O.samples == cfg['iters'] * cfg['B']


def test_oracle_q_values_against_the_reference_dueling_head(golden):
    g = golden('dqn_qnet')
    x = torch.from_numpy(g['x']).double()
    for tag in ('noduel', 'duel'):
        a = [(w.double(), b.double()) for w, b in golden_layers(g, tag + '/model/', 'action')]
        s = golden_layers(g, tag + '/model/', 'state')
        s = [(w.double(), b.double()) for w, b in s] if s is not None else None
        q = odqn.q_values(x, a, s)
        assert np.abs(q.numpy() - g[tag + '/q']).max() <= 1e-5


@pytest.mark.parametrize('sched', ['linear', 'piecewise'])
def test_exploration_against_the_reference_agent(golden, sched):
    """QAgent.act's branch on the reference's own draws: greedy when u > eps, else the uniform draw; epsilon from the
    schedule at T (this engine explores when u < eps: the two differ only at u == eps exactly)."""
    from surreal_b200.agent.q_agent import exploration_schedule
    from surreal_b200.session import Config
    g = golden('dqn_explore')
    S = exploration_schedule(Config(json.loads(str(g[sched + '/exploration']))))
    a = [(w.double(), b.double()) for w, b in golden_layers(g, sched + '/model/', 'action')]
    s = [(w.double(), b.double()) for w, b in golden_layers(g, sched + '/model/', 'state')]
    q = odqn.q_values(torch.from_numpy(g[sched + '/x']).double(), a, s).numpy()
    rows = g[sched + '/rows']
    explored = 0
    for T, eps, u, ra, act in rows:
        assert S.value(int(T)) == eps
        assert u != eps
        if u < eps:
            explored += 1
            assert act == ra
        else:
            assert ra == -1 and act == q[int(T)].argmax()
    assert 0 < explored < len(rows)

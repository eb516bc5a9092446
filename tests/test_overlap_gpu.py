"""The learner beside the rollout: PipelinedEngine gives the learner the SMs the one-wave rollout leaves free as a grid budget
(PPOLearner.set_sm_budget).  The learner's persistent kernels must compute the same bits at any grid: the epoch kernel
(csrc/epoch2.cu) sizes its row split and squared-norm chunks for one CTA per SM whatever grid it gets, and the critic pass
(csrc/mlp_fwd_tc5.cu) keeps its tiles.  So the overlapped engine and the old head | wait | epochs schedule end in the same
state."""
import numpy as np
import pytest
import torch

from helpers import ppo_configs
from test_epoch_kernel_gpu import CASES, _batch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _learner_state(L):
    return [L.model.actor.params, L.model.critic.params, L.actor_optim.exp_avg, L.actor_optim.exp_avg_sq,
            L.critic_optim.exp_avg, L.critic_optim.exp_avg_sq, L._stats] + \
        ([L.model.z_stats] if L.model.z_stats is not None else [])


# clip and adapt at the bench's layer sizes, and the two ragged shapes (rows, widths and heads off every tile boundary)
@pytest.mark.parametrize('case', [2, 3, 4, 5])
def test_epoch_kernel_is_bit_identical_at_any_grid(case, monkeypatch):
    from surreal_b200.learner import PPOLearner
    monkeypatch.setenv('SB200_EPOCH_KERNEL', '2')
    kw = CASES[case]
    res = {}
    for grid in (0, 68, 37):
        torch.manual_seed(11)
        lc, ec, sc = ppo_configs(**kw)
        L = PPOLearner(lc, ec, sc)
        L.set_sm_budget(grid)
        epochs = []
        for it in range(3):
            L.learn(_batch(kw['B'], kw['n_step'], kw['D'], kw['A'], seed=10 * case + it))
            epochs.append(L.last_n_policy_epochs)
        torch.cuda.synchronize()
        assert L._ek is not None and L._ek[3] is not None, 'the one-launch kernel was not the path taken'
        assert L._ek[3].plan(L._ek[1], L._ek[2])['grid'] == (grid or min(_n_sm(), 192))
        res[grid] = (epochs, [t.clone() for t in _learner_state(L)])
    for grid in (68, 37):
        assert res[grid][0] == res[0][0], (grid, res[grid][0], res[0][0])
        for i, (a, b) in enumerate(zip(res[0][1], res[grid][1])):
            assert torch.equal(a, b), 'grid %d: state tensor %d differs from the full grid' % (grid, i)


@pytest.mark.parametrize('dims,rows', [([64, 256, 256, 1], 1024 * 129), ([32, 128, 64, 3], 19205)])
def test_critic_pass_is_bit_identical_at_a_capped_grid(dims, rows):
    from surreal_b200 import ops
    gen = torch.Generator().manual_seed(rows)
    acts = [ops.ACT_RELU, ops.ACT_RELU, ops.ACT_TANH if dims[-1] > 1 else ops.ACT_NONE]
    net = ops.FlatNet(dims, acts, DEV)
    net.params.copy_((torch.randn(net.params.numel(), generator=gen) * 0.1).to(DEV))
    x = (torch.randn(rows, dims[0], generator=gen) * 2 + 0.5).to(DEV)
    f = ops.Tc5Forward(net)
    assert f.supported(rows)
    outs = []
    for grid in (0, 68, 37):
        f.grid = grid
        out = torch.full((rows, dims[-1]), float('nan'), device=DEV)
        f(x, out)
        outs.append(out)
    torch.cuda.synchronize()
    assert not torch.isnan(outs[0]).any()
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def _engine(overlap, steps):
    from surreal_b200.launch import SurrealDefaultLauncher, PipelinedEngine
    from surreal_b200.agent import PPOAgent
    from surreal_b200.learner import PPOLearner
    from surreal_b200.replay import FIFOReplay
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    N, n, D, A = 1024, 128, 64, 8                      # the bench shape: the rollout runs in one wave on 64 SMs
    torch.manual_seed(0)
    np.random.seed(0)
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=(256, 256), critic_h=(256, 256), n_step=n, stride=n, B=N,
                             memory_size=2 * N, exp_interval=N)
    make_synthetic_env_config(ec, N, D, A, seed=3)
    ec.limit_episode_length = 2 * n
    sc.agent.fetch_parameter_interval = n
    lc.parameter_publish.min_publish_interval = 0.0
    la = SurrealDefaultLauncher(PPOAgent, PPOLearner, FIFOReplay, sc, ec, lc)
    agent, replay, learner = la.setup_engine()
    agent.set_noise(np.random.default_rng(1000).uniform(-0.5, 0.5, N))
    if not overlap:
        agent.rollout_footprint = lambda: 0             # what a rollout in several waves reports: the hook schedule
    eng = PipelinedEngine(agent, replay, learner, n)
    assert eng.overlap == overlap
    assert learner.sm_budget == (_n_sm() - agent.rollout_footprint() if overlap else 0)
    assert (learner.before_epochs_hook is None) == overlap
    eng.prime()
    for _ in range(steps):
        eng.step()
    eng.drain()
    state = [t.clone() for t in _learner_state(learner)]
    fifo = [getattr(replay, k).clone() for k in ('r_obs', 'r_act', 'r_pd', 'r_rew', 'r_done')]
    return state, fifo, list(learner.epoch_history)


def test_overlapped_engine_matches_the_hook_schedule():
    from surreal_b200.agent import PPOAgent  # noqa: F401
    st_o, fifo_o, ep_o = _engine(True, 5)
    st_h, fifo_h, ep_h = _engine(False, 5)
    assert ep_o == ep_h
    for i, (a, b) in enumerate(zip(st_o, st_h)):
        assert torch.equal(a, b), 'learner state tensor %d differs' % i
    for i, (a, b) in enumerate(zip(fifo_o, fifo_h)):
        assert torch.equal(a, b), 'FIFO array %d differs' % i

"""DDPGLearner / DDPGAgent (CUDA) vs goldens produced by the reference's own DDPGLearner._optimize / DDPGAgent.act."""
import numpy as np
import pytest
import torch

from helpers import ddpg_configs, ref_state_dict

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('tag', ['hard', 'soft_clipcritic'])
def test_ddpg_optimize_matches_reference(golden, tag):
    from surreal_b200.learner import DDPGLearner
    g = golden('ddpg_optimize_' + tag)
    cfg, stats = g.js('cfg'), g.js('stats')
    lc, ec, sc = ddpg_configs(D=cfg['D'], A=cfg['A'], actor_h=cfg['actor_h'], critic_h=cfg['critic_h'], B=cfg['B'],
                              n_step=cfg['n_step'], target=cfg['target'], clip_critic=cfg['clip_critic'],
                              lr_actor=cfg['lr_actor'], lr_critic=cfg['lr_critic'])
    L = DDPGLearner(lc, ec, sc)
    L.model.load_state_dict(ref_state_dict(g.sub('init/model/')))
    L.model_target.load_state_dict(ref_state_dict(g.sub('init/target/')))
    for it in range(3):
        b = g.sub('it%d/' % it)
        st = L.learn({'obs': {'low_dim': {'flat_inputs': b['obs']}}, 'obs_next': {'low_dim': {'flat_inputs': b['obs_next']}},
                      'actions': b['actions'], 'rewards': b['rewards'], 'dones': b['dones']})
        torch.cuda.synchronize()
        for k, v in stats[it].items():
            assert abs(st[k] - v) <= 1e-5 * max(1.0, abs(v)), '%s it%d: got %.9g expected %.9g' % (k, it, st[k], v)
        for name, model in (('model', L.model), ('target', L.model_target)):
            exp = ref_state_dict(g.sub('it%d/%s/' % (it, name)))
            got = model.state_dict()
            for k, e in exp.items():
                d = float((got[k].cpu().reshape(e.shape) - e).abs().max())
                assert d <= 2e-5, '%s %s it%d drift %.3e' % (name, k, it, d)      # lr_critic = 1e-3: 2% of one step


@pytest.mark.parametrize('tag', ['td3_double', 'td3_double_reg'])
def test_ddpg_td3_options_match_reference(golden, tag):
    """use_double_critic / use_action_regularization (ddpg.py:267-283,298-321) against goldens produced by the
    reference: y = min over two target critics, the smoothing noise reaches only critic 2, critic_loss reports
    critic 2's loss, both critics and target2 follow the reference's parameters."""
    from surreal_b200.learner import DDPGLearner
    g = golden('ddpg_optimize_' + tag)
    cfg, stats = g.js('cfg'), g.js('stats')
    lc, ec, sc = ddpg_configs(D=cfg['D'], A=cfg['A'], actor_h=cfg['actor_h'], critic_h=cfg['critic_h'], B=cfg['B'],
                              n_step=cfg['n_step'], target=cfg['target'], clip_critic=cfg['clip_critic'],
                              lr_actor=cfg['lr_actor'], lr_critic=cfg['lr_critic'])
    lc.algo.network.use_double_critic = True
    lc.algo.network.use_action_regularization = bool(cfg['action_regularization'])
    L = DDPGLearner(lc, ec, sc)
    L.model.load_state_dict(ref_state_dict(g.sub('init/model/')))
    L.model_target.load_state_dict(ref_state_dict(g.sub('init/target/')))
    L.model2.load_state_dict(ref_state_dict(g.sub('init/model2/')))
    L.model_target2.load_state_dict(ref_state_dict(g.sub('init/target2/')))
    for it in range(3):
        b = g.sub('it%d/' % it)
        if cfg['action_regularization']:                       # N(0, 0.2) draws of the fixture -> unit draws
            L.policy_noise_draws = torch.tensor(b['policy_noise_unclipped'] / 0.2, dtype=torch.float32, device='cuda')
        st = L.learn({'obs': {'low_dim': {'flat_inputs': b['obs']}}, 'obs_next': {'low_dim': {'flat_inputs': b['obs_next']}},
                      'actions': b['actions'], 'rewards': b['rewards'], 'dones': b['dones']})
        torch.cuda.synchronize()
        for k, v in stats[it].items():
            assert abs(st[k] - v) <= 1e-5 * max(1.0, abs(v)), '%s it%d: got %.9g expected %.9g' % (k, it, st[k], v)
        for name, model in (('model', L.model), ('model2', L.model2), ('target', L.model_target),
                            ('target2', L.model_target2)):
            exp = ref_state_dict(g.sub('it%d/%s/' % (it, name)))
            got = model.state_dict()
            for k, e in exp.items():
                d = float((got[k].cpu().reshape(e.shape) - e).abs().max())
                assert d <= 2e-5, '%s %s it%d drift %.3e' % (name, k, it, d)


def test_ddpg_agent_act_matches_reference(golden):
    from surreal_b200.agent import DDPGAgent
    g = golden('ddpg_act')
    N = len(g['obs'])
    lc, ec, sc = ddpg_configs(D=9, A=3)
    ec.num_envs = N
    ec.num_agents = 4
    ag = DDPGAgent(lc, ec, sc, 0, 'training')
    ag.model.load_state_dict(ref_state_dict(g.sub('model/')))
    ag._sigma.fill_(float(g['sigma']))                       # every row of the fixture is agent 3 of 4
    a = ag.act({'low_dim': {'flat_inputs': g['obs']}}, unit_noise=g['unit_noise'])
    assert a.dtype == np.float32
    np.testing.assert_allclose(a, g['actions'], rtol=0, atol=2e-6)
    assert ag.sigma.tolist() == [0.0, 0.25, 0.5, 0.75, 1.0][:N] or N != 5


def test_ddpg_agent_ou_noise_matches_reference(golden):
    """noise_type 'ou_noise': the float64 Ornstein-Uhlenbeck walk of the reference (one actor, 8 steps, reset by
    pre_episode after 5) replayed with the same unit draws; several actors keep independent states."""
    from surreal_b200.agent import DDPGAgent
    g = golden('ddpg_act_ou')
    lc, ec, sc = ddpg_configs(D=9, A=3)
    lc.algo.exploration.noise_type = 'ou_noise'
    lc.algo.exploration.theta, lc.algo.exploration.dt = float(g['theta']), float(g['dt'])
    ec.num_envs, ec.num_agents = 2, 4
    ag = DDPGAgent(lc, ec, sc, 0, 'training')
    ag.model.load_state_dict(ref_state_dict(g.sub('model/')))
    ag._sigma64.fill_(float(g['sigma']))                     # both rows replay agent 3 of 4 of the fixture
    for i in range(len(g['obs'])):
        if i == int(g['reset_at']):
            ag.pre_episode()
        obs2 = np.stack([g['obs'][i], g['obs'][i]])
        un = np.stack([g['unit_noise'][i], -g['unit_noise'][i]])              # second actor: mirrored draws
        a = ag.act({'low_dim': {'flat_inputs': obs2}}, unit_noise=un)
        np.testing.assert_allclose(a[0], g['actions'][i], rtol=0, atol=2e-6)
        st = ag._ou_state.cpu().numpy()
        np.testing.assert_allclose(st[0], g['ou_states'][i], rtol=0, atol=1e-7)
        np.testing.assert_allclose(st[1], -g['ou_states'][i], rtol=0, atol=1e-7)
    ag.agent_mode = 'eval_deterministic'
    before = ag._ou_state.clone()
    ag.act({'low_dim': {'flat_inputs': obs2}})
    assert torch.equal(before, ag._ou_state)                 # deterministic evaluation does not advance the walk


def test_ddpg_engine_end_to_end():
    """actors -> n-step SSAR staging -> UniformReplay ring -> CPython-exact sampling -> DDPGLearner."""
    import random
    from surreal_b200.launch import SurrealDefaultLauncher
    from surreal_b200.agent import DDPGAgent
    from surreal_b200.learner import DDPGLearner
    from surreal_b200.replay import UniformReplay
    from surreal_b200.main.ppo_configs import make_synthetic_env_config
    N = 32
    lc, ec, sc = ddpg_configs(D=12, A=4, actor_h=(48, 32), critic_h=(64, 48), B=64, n_step=3, memory_size=500, start=100)
    make_synthetic_env_config(ec, N, 12, 4, seed=1)
    ec.num_agents = N
    ec.limit_episode_length = 20
    la = SurrealDefaultLauncher(DDPGAgent, DDPGLearner, UniformReplay, sc, ec, lc)
    agent, replay, learner = la.setup_engine()
    agent.main_loop(max_steps=30)
    torch.cuda.synchronize()
    # every actor emits from its (n_step)-th step of an episode on: 20-step episodes -> 18 per episode
    per_actor = 18 + (30 - 20 - 2)
    assert len(replay) == min(500, N * per_actor)
    assert replay.start_sample_condition()
    random.seed(5)
    expect_idx = [random.randint(0, len(replay) - 1) for _ in range(64)]
    random.seed(5)
    batch = replay.sample(64)
    assert batch['indices'].tolist() == expect_idx
    assert torch.equal(batch['actions'].cpu(), replay.r_act[torch.tensor(expect_idx)].cpu())
    st = learner.learn(batch)
    for k in ['actor_loss', 'critic_loss', 'Q_target', 'Q_policy', 'action_norm', 'rewards']:
        assert np.isfinite(st[k])
    assert float(replay.r_act.abs().max()) <= 1.0


def test_ddpg_out_of_range_actions_leave_state_untouched():
    """The reference asserts |a| <= 1 BEFORE any update (ddpg.py:261-262), and a NaN action fails it too.  Here the whole update is one graph, so the
    target kernel raises a device flag that turns every optimiser / soft-update kernel of that learn() into a no-op:
    the AssertionError must leave actor, critic, targets and Adam moments bit-identical."""
    from surreal_b200.learner import DDPGLearner
    lc, ec, sc = ddpg_configs(D=9, A=3, B=16, target={'type': 'soft', 'tau': 0.01, 'interval': 1})
    L = DDPGLearner(lc, ec, sc)
    rng = np.random.default_rng(0)
    mk = lambda amax: {'obs': {'low_dim': {'flat_inputs': rng.standard_normal((16, 9)).astype(np.float32)}},   # noqa: E731
                       'obs_next': {'low_dim': {'flat_inputs': rng.standard_normal((16, 9)).astype(np.float32)}},
                       'actions': (rng.uniform(-1, 1, (16, 3)) * amax).astype(np.float32),
                       'rewards': rng.standard_normal((16, 1)), 'dones': np.zeros((16, 1))}
    L.learn(mk(1.0))                                            # a good batch first (captures the graph, moves Adam)
    snap = [t.clone() for t in (L.model.actor.params, L.model.critic.params, L.model_target.actor.params,
                                L.model_target.critic.params, L.actor_optim.exp_avg, L.critic_optim.exp_avg_sq)]
    nan_batch = mk(1.0)
    nan_batch['actions'][9, 2] = np.nan                         # torch.max propagates NaN: the reference rejects it
    for bad in (mk(3.0), nan_batch):
        with pytest.raises(AssertionError):
            L.learn(bad)
        torch.cuda.synchronize()
        for a, b in zip(snap, (L.model.actor.params, L.model.critic.params, L.model_target.actor.params,
                               L.model_target.critic.params, L.actor_optim.exp_avg, L.critic_optim.exp_avg_sq)):
            assert torch.equal(a, b)
    before = L.model.critic.params.clone()
    L.learn(mk(1.0))                                            # and the learner keeps working afterwards
    assert not torch.equal(before, L.model.critic.params)

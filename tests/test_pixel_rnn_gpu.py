"""CNN + LSTM policy (pixel input with algo.rnn.if_rnn_policy -- the reference's default PPO config on a camera env):
uint8 frame -> CNN stem -> LSTM stem -> heads (ppo_net.py:143-156,268-279; builders.py:23-33).

  * PPOLearner.learn + publish against goldens produced by the REFERENCE's PPOLearner, graph == eager bit for bit;
  * PPOAgent.act against the reference's act (cells handed off, reset) and against a float64 step at scale;
  * window records of host and device pixel envs, the wide-row commit kernel, FIFO sample of frames + cells;
  * checkpoints with the optimiser state (pixel + LSTM and pixel-only), and a reference-written one."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import ppo_configs, ref_state_dict

pytestmark = pytest.mark.gpu

LOSS_STATS = ['_surr_loss', '_clip_surr_loss', '_kl_loss_adapt', '_entropy', '_pol_kl', '_val_loss', '_avg_return_targ',
              '_avg_log_sig', '_avg_behave_likelihood', '_avg_is_weight', '_ref_behave_diff']


def _cfg(C, HW, F_, A, actor_h, critic_h, n, B, mode, lr, exp_interval, horizon, rnn_hidden, rnn_layer, N=None):
    lc, ec, sc = ppo_configs(D=1, A=A, actor_h=actor_h, critic_h=critic_h, n_step=n, stride=n, B=B, mode=mode, lr=lr,
                             exp_interval=exp_interval, use_z=False)
    ec.obs_spec = {'pixel': {'camera0': (C, HW, HW)}}
    ec.pixel_input = True
    lc.model.cnn_feature_dim = F_
    lc.algo.rnn.if_rnn_policy = True
    lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = horizon, rnn_hidden, rnn_layer
    if N is not None:
        ec.num_envs = N
    return lc, ec, sc


def _gcfg(cfg, **kw):
    a = dict(C=cfg['C'], HW=cfg['HW'], F_=cfg['cnn_feature_dim'], A=cfg['A'], actor_h=cfg['actor_h'], critic_h=cfg['critic_h'],
             n=cfg['n_step'], B=cfg['B'], mode=cfg.get('mode', 'clip'), lr=cfg['lr'], exp_interval=cfg['exp_interval'],
             horizon=cfg['horizon'], rnn_hidden=cfg['rnn_hidden'], rnn_layer=cfg['rnn_layer'])
    a.update(kw)
    return _cfg(**a)


def _batch(b):
    return {'obs': {'pixel': {'camera0': b['obs']}}, 'obs_next': {'pixel': {'camera0': b['obs_next']}}, 'actions': b['actions'],
            'rewards': b['rewards'], 'dones': b['dones'], 'persistent_infos': [b['pd']], 'onetime_infos': [b['h0'], b['c0']]}


@pytest.mark.parametrize('tag', ['pixel_rnn_clip', 'pixel_rnn_adapt', 'pixel_rnn2_clip'])
def test_ppo_learn_pixel_rnn_matches_reference(golden, tag):
    from surreal_b200.learner import PPOLearner
    g = golden('ppo_learn_' + tag)
    cfg, hyper, stats = g.js('cfg'), g.js('hyper'), g.js('stats')
    L = PPOLearner(*_gcfg(cfg))
    L.model.load_state_dict(ref_state_dict(g.sub('init/')))
    L.ref_target_model.update_target_params(L.model)
    lr = cfg['lr']
    for it in range(cfg['iters']):
        b = g.sub('it%d/' % it)
        st = L.learn(_batch(b))
        L.publish_parameter(it, message='')
        torch.cuda.synchronize()
        assert L.last_n_policy_epochs == hyper[it]['n_policy_epochs']
        assert float((L._adv.cpu() - torch.tensor(b['adv'])).abs().max()) <= 1e-5
        rms = float(np.sqrt((b['ret'] ** 2).mean()))
        assert float((L._ret.cpu() - torch.tensor(b['ret'])).abs().max()) <= 1e-5 * max(1.0, rms)
        for k, v in stats[it].items():
            assert k in st, k
            tol = 1e-5 * max(1.0, abs(v)) if k in LOSS_STATS else 2e-4 * max(1.0, abs(v))
            if k == '_val_explained_var':
                tol = 1e-4
            assert abs(st[k] - v) <= tol, '%s it%d: got %.9g expected %.9g' % (k, it, st[k], v)
        after = ref_state_dict(g.sub('it%d/after/' % it))
        got = L.model.state_dict()
        assert set(after) == set(got), sorted(set(after) ^ set(got))
        worst, key = max((float((got[k].cpu().reshape(e.shape) - e).abs().max()), k) for k, e in after.items())
        assert worst <= max(2e-6, 0.02 * lr), 'params drifted by %.3e (%s)' % (worst, key)
        if cfg['mode'] == 'clip':
            assert L.clip_epsilon == pytest.approx(hyper[it]['clip_epsilon'], rel=1e-12)
        else:
            assert L.beta == pytest.approx(hyper[it]['beta'], rel=1e-12)
    if cfg['mode'] == 'adapt':
        assert min(h['n_policy_epochs'] for h in hyper) < cfg['epoch_policy']          # the KL early stop fired


def _snapshot(L):
    m = L.model
    return [m.actor.params, m.critic.params, m.cnn_stem.params, m.rnn_stem.params, L.actor_rnn.exp_avg, L.critic_rnn.exp_avg_sq,
            L.actor_stem.exp_avg, L.actor_stem.exp_avg_sq, L.critic_stem.exp_avg, L.critic_stem.exp_avg_sq,
            L.actor_optim.exp_avg_sq, L.critic_optim.exp_avg_sq, L.ref_target_model.cnn_stem.params,
            L.ref_target_model.rnn_stem.params]


@pytest.mark.parametrize('tag', ['pixel_rnn_adapt', 'pixel_rnn2_clip'])
def test_graph_and_eager_learn_are_bit_identical(golden, tag):
    from surreal_b200.learner import PPOLearner
    g = golden('ppo_learn_' + tag)
    cfg = g.js('cfg')
    runs = []
    for graph in (True, False):
        L = PPOLearner(*_gcfg(cfg))
        L.use_cuda_graph = graph
        L.model.load_state_dict(ref_state_dict(g.sub('init/')))
        L.ref_target_model.update_target_params(L.model)
        sts = []
        for it in range(cfg['iters']):
            sts.append(L.learn(_batch(g.sub('it%d/' % it))))
            L.publish_parameter(it, message='')
        torch.cuda.synchronize()
        runs.append((sts, [t.clone() for t in _snapshot(L)]))
    assert runs[0][0] == runs[1][0]
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)


def _agent(N, C, HW, F_, A, H, layers, actor_h=(64, 48), critic_h=(64, 48)):
    from surreal_b200.agent import PPOAgent
    lc, ec, sc = _cfg(C, HW, F_, A, list(actor_h), list(critic_h), 4, 4, 'clip', 1e-4, 64, 2, H, layers, N=N)
    return PPOAgent(lc, ec, sc, 0, 'training'), (lc, ec, sc)


def test_ppo_agent_act_pixel_rnn_matches_reference(golden):
    """One actor, seven single frames (numpy in): onetime_infos (1, H) = the cells BEFORE the step, reset() at step 4."""
    g = golden('ppo_act_pixel_rnn')
    Hd = int(g['rnn_hidden'])
    ag, _ = _agent(1, int(g['C']), int(g['HW']), int(g['cnn_feature_dim']), 3, Hd, 1, actor_h=(32, 24), critic_h=(28, 20))
    ag.model.load_state_dict(ref_state_dict(g.sub('model/')))
    ag.set_noise(np.array([float(g['noise'])]))
    for i in range(len(g['obs'])):
        if i == int(g['reset_at']):
            ag.reset()
        a, info = ag.act({'pixel': {'camera0': g['obs'][i]}}, eps=g['eps'][i])
        np.testing.assert_allclose(np.asarray(info[0][0]).reshape(-1), g['h_before'][i].reshape(-1), rtol=0, atol=2e-6)
        np.testing.assert_allclose(np.asarray(info[0][1]).reshape(-1), g['c_before'][i].reshape(-1), rtol=0, atol=2e-6)
        np.testing.assert_allclose(info[1][0], g['pds'][i], rtol=0, atol=2e-6)
        np.testing.assert_allclose(a, g['actions'][i], rtol=0, atol=5e-6)


def _f64_step(sd, layers, frames, h, c):
    """float64 CNN -> LSTM (one step from h / c [L, N, H]) -> actor mean."""
    d = {k: v.detach().double().cpu() for k, v in sd.items()}
    x = frames.double().cpu() / 255.0
    x = torch.relu(F.conv2d(x, d['cnn_stem.model.seq.0.weight'], d['cnn_stem.model.seq.0.bias'], stride=4))
    x = torch.relu(F.conv2d(x, d['cnn_stem.model.seq.2.weight'], d['cnn_stem.model.seq.2.bias'], stride=2)).flatten(1)
    x = torch.relu(F.linear(x, d['cnn_stem.model.seq.5.weight'], d['cnn_stem.model.seq.5.bias']))
    hs, cs = [], []
    for k in range(layers):
        gates = F.linear(x, d['rnn_stem.weight_ih_l%d' % k], d['rnn_stem.bias_ih_l%d' % k]) + \
            F.linear(h[k].double().cpu(), d['rnn_stem.weight_hh_l%d' % k], d['rnn_stem.bias_hh_l%d' % k])
        i, f, gg, o = gates.chunk(4, 1)
        cn = torch.sigmoid(f) * c[k].double().cpu() + torch.sigmoid(i) * torch.tanh(gg)
        x = torch.sigmoid(o) * torch.tanh(cn)
        hs.append(x)
        cs.append(cn)
    for l in range(3):
        x = F.linear(x, d['actor.model.seq.%d.weight' % (2 * l)], d['actor.model.seq.%d.bias' % (2 * l)])
        x = torch.relu(x) if l < 2 else torch.tanh(x)
    return x, torch.stack(hs), torch.stack(cs)


@pytest.mark.parametrize('N,host', [(256, False), (256, True), (1024, False), (1024, True)])
def test_ppo_agent_act_pixel_rnn_at_scale(N, host):
    """[4, 84, 84] frames, LSTM(100), 20 steps with injected eps: each step's onetime_infos are the cells held before
    it, pd and the new cells match one float64 step from those cells, and a free-running float64 trajectory stays close."""
    A, H, steps = 6, 100, 20
    ag, _ = _agent(N, 4, 84, 84, A, H, 1)
    ag._rnn_state()
    gen = torch.Generator().manual_seed(N)
    sd = ag.model.state_dict()
    h64 = torch.zeros(1, N, H, dtype=torch.float64)
    c64 = torch.zeros_like(h64)
    drift = 0.0
    for t in range(steps):
        fr = torch.randint(0, 256, (N, 4, 84, 84), generator=gen, dtype=torch.uint8)
        eps = torch.randn(N, A, generator=gen).numpy()
        obs = fr.numpy() if host else fr.cuda()
        h_b, c_b = ag._hs.clone(), ag._cs.clone()
        a, info = ag.act({'pixel': {'camera0': obs}}, eps=eps)
        oh = torch.as_tensor(np.asarray(info[0][0].cpu() if torch.is_tensor(info[0][0]) else info[0][0]))
        assert torch.equal(oh.transpose(0, 1).cpu(), h_b.cpu())
        mean, hn, cn = _f64_step(sd, 1, fr, h_b, c_b)
        pd = torch.as_tensor(np.asarray(info[1][0].cpu() if torch.is_tensor(info[1][0]) else info[1][0]))
        assert float((pd[:, :A].double() - mean).abs().max()) <= 2.5e-6
        assert float((ag._hs.double().cpu() - hn).abs().max()) <= 2.5e-6
        assert float((ag._cs.double().cpu() - cn).abs().max()) <= 2.5e-6
        _, h64, c64 = _f64_step(sd, 1, fr, h64, c64)
        drift = max(drift, float((ag._hs.double().cpu() - h64).abs().max()))
    assert drift <= 1.5e-5, drift


class _HostPixelEnv:
    """A batched HOST env (numpy in / numpy out) replaying a device SyntheticPixelEnv's frames."""

    def __init__(self, env):
        self.env, self.N, self.D, self.A = env, env.N, env.D, env.A
        self.step_counter = env.step_counter        # the same Philox step counter as the device env's run

    def reset(self):
        obs, info = self.env.reset()
        return {'pixel': {'camera0': obs['pixel']['camera0'].cpu().numpy()}}, info

    def step(self, a):
        obs, r, d, info = self.env.step(torch.as_tensor(np.asarray(a), dtype=torch.float32, device='cuda'))
        info = {'obs_next': {'pixel': {'camera0': info['obs_next']['pixel']['camera0'].cpu().numpy()}}}
        return {'pixel': {'camera0': obs['pixel']['camera0'].cpu().numpy()}}, r.cpu().numpy(), d.cpu().numpy(), info


def _run_records(N, host, wide, C=2, HW=20, steps=11, H=6, layers=2):
    from surreal_b200.agent import PPOAgent
    from surreal_b200.env import SyntheticPixelEnv
    from surreal_b200.replay import FIFOReplay
    n = 4
    lc, ec, sc = _cfg(C, HW, 12, 3, [32, 24], [28, 20], n, N, 'clip', 1e-4, 64, 2, H, layers, N=N)
    lc.algo.stride = 2
    lc.replay.memory_size = 2 * N              # windows drop at capacity
    torch.manual_seed(3)
    R = FIFOReplay(lc, ec, sc)
    ag = PPOAgent(lc, ec, sc, 0, 'training')
    ag.set_noise(np.linspace(-0.2, 0.2, N))
    env = SyntheticPixelEnv(N, (C, HW, HW), 3, limit_episode_length=5, seed=9)
    ag.env = w = ag.prepare_env_agent(_HostPixelEnv(env) if host else env)
    w.wide_commit = wide
    obs, _ = w.reset()
    for t in range(steps):
        a = ag.act(obs)
        obs, _, _, _ = w.step(a)
        if t == 3:
            env.ep_step[::3] = 3                   # staggered episode ends
    torch.cuda.synchronize()
    return R, w


@pytest.mark.parametrize('N', [1, 7, 256])
def test_host_and_device_pixel_envs_write_identical_records(N):
    """Frame words and [h | c] cells of every staged row and FIFO record: host env == device env == the wide-row commit
    kernel (rows small enough for the shared-memory kernel too)."""
    runs = [_run_records(N, host, wide) for host, wide in ((False, False), (True, False), (False, True))]
    ref = runs[0]
    for R, w in runs[1:]:
        for name in ('r_obs', 'r_act', 'r_pd', 'r_rew', 'r_done', 'state'):
            assert torch.equal(getattr(R, name).view(torch.int32) if getattr(R, name).dtype == torch.float32 else getattr(R, name),
                               getattr(ref[0], name).view(torch.int32) if getattr(ref[0], name).dtype == torch.float32
                               else getattr(ref[0], name)), name
        assert torch.equal(w.stage_obs.view(torch.int32), ref[1].stage_obs.view(torch.int32))
    if N == 256:
        assert ref[0]._read_state()['dropped'] > 0


def test_sample_returns_frames_and_cells():
    """FIFO sample of pixel + LSTM windows: uint8 frames and onetime_infos [B, L, H] = the cells the actor held at the
    window's first step; host insert with onetime_infos round-trips and rejects the wrong cell count."""
    from surreal_b200.replay import FIFOReplay
    C, HW, n, L_, H, A = 2, 20, 3, 2, 5, 3
    lc, ec, sc = _cfg(C, HW, 12, A, [8], [8], n, 2, 'clip', 1e-4, 64, 2, H, L_)
    R = FIFOReplay(lc, ec, sc)
    rng = np.random.default_rng(0)
    wins = []
    for _ in range(2):
        fr = rng.integers(0, 256, size=(n + 1, C, HW, HW), dtype=np.uint8)
        hc = [rng.standard_normal((L_, H)).astype(np.float32), rng.standard_normal((L_, H)).astype(np.float32)]
        exp = dict(obs=[{'pixel': {'camera0': fr[t]}} for t in range(n)], obs_next={'pixel': {'camera0': fr[n]}},
                   actions=[np.zeros(A)] * n, rewards=[0.0] * n, dones=[0.0] * n,
                   persistent_infos=[[np.zeros(2 * A, dtype=np.float32)]] * n, onetime_infos=hc)
        R.insert(exp)
        wins.append((fr, hc))
    bad = dict(exp, onetime_infos=[np.zeros((1, H), np.float32), np.zeros((1, H), np.float32)])
    with pytest.raises(ValueError):
        R.insert(bad)
    b = R.sample(2)
    for i, (fr, hc) in enumerate(wins):
        got = torch.cat([b['obs']['pixel']['camera0'][i], b['obs_next']['pixel']['camera0'][i]]).cpu().numpy()
        assert np.array_equal(got, fr)
        assert tuple(b['onetime_infos'][0].shape) == (2, L_, H)
        assert np.array_equal(b['onetime_infos'][0][i].cpu().numpy(), hc[0])
        assert np.array_equal(b['onetime_infos'][1][i].cpu().numpy(), hc[1])


def test_frame_gather_is_bit_exact():
    """The learner's frame gather (rows_zfilter without a filter) copies frame bytes whose words are denormal / NaN floats."""
    from surreal_b200.model.lstm_stem import rows_zfilter
    B, n1, od, D = 3, 4, 64, 80
    src = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, n1, D), dtype=torch.int32)
    src[0, 0, :4] = torch.tensor([1, 0x7fc00001, 0x7f800001, -1], dtype=torch.int32)     # denormal, qNaN / sNaN payloads
    x = src.cuda().view(torch.float32)
    out = torch.zeros(B * n1, od, device='cuda')
    rows_zfilter(x, D, n1 * D, B, n1, od, None, 0.0, out)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32).cpu(), src[:, :, :od].reshape(B * n1, od))


def _ckpt_roundtrip(tmp_path, lc, ec, sc, batches):
    from surreal_b200.learner import PPOLearner

    def make(folder, restore_from=None):
        import copy
        from surreal_b200.session import Config
        sc2 = Config(copy.deepcopy(sc.to_dict()))
        sc2.folder = str(folder)
        sc2.checkpoint.learner.periodic = 1
        sc2.checkpoint.learner.min_interval = 0
        sc2.checkpoint.learner.include_optimizer = True
        if restore_from is not None:
            sc2.checkpoint.restore = True
            sc2.checkpoint.restore_folder = str(restore_from)
        return PPOLearner(lc, ec, sc2)
    torch.manual_seed(5)
    A_ = make(tmp_path / 'a')
    for it, b in enumerate(batches[:-1]):
        A_.learn(b)                                   # saves the checkpoint
        if it < len(batches) - 2:
            A_.publish_parameter(it)
    torch.manual_seed(555)
    B_ = make(tmp_path / 'b', restore_from=tmp_path / 'a')
    sa, sb = A_.learn(batches[-1]), B_.learn(batches[-1])
    torch.cuda.synchronize()
    assert sa == sb
    for k, v in A_.model.state_dict().items():
        assert torch.equal(v, B_.model.state_dict()[k]), k
    for t in ('actor_stem', 'critic_stem'):
        for m in ('exp_avg', 'exp_avg_sq'):
            assert torch.equal(getattr(getattr(A_, t), m), getattr(getattr(B_, t), m)), (t, m)


def test_pixel_rnn_learner_checkpoint_continues_bit_identically(tmp_path, golden):
    g = golden('ppo_learn_pixel_rnn_clip')
    cfg = g.js('cfg')
    bs = [_batch(g.sub('it%d/' % it)) for it in range(2)]
    _ckpt_roundtrip(tmp_path, *_gcfg(cfg), bs + [bs[0]])


def test_pixel_learner_checkpoint_continues_bit_identically(tmp_path, golden):
    """Pixel-only learner with include_optimizer: both optimisers' Adam moments over the CNN stem are saved too."""
    g = golden('ppo_learn_pixel_clip')
    cfg = g.js('cfg')
    lc, ec, sc = ppo_configs(D=1, A=cfg['A'], actor_h=cfg['actor_h'], critic_h=cfg['critic_h'], n_step=cfg['n_step'],
                             stride=cfg['n_step'], B=cfg['B'], mode=cfg['mode'], lr=cfg['lr'], exp_interval=cfg['exp_interval'],
                             use_z=False)
    ec.obs_spec = {'pixel': {'camera0': (cfg['C'], cfg['HW'], cfg['HW'])}}
    ec.pixel_input = True
    lc.model.cnn_feature_dim = cfg['cnn_feature_dim']
    bs = []
    for it in range(2):
        b = g.sub('it%d/' % it)
        bs.append({'obs': {'pixel': {'camera0': b['obs']}}, 'obs_next': {'pixel': {'camera0': b['obs_next']}},
                   'actions': b['actions'], 'rewards': b['rewards'], 'dones': b['dones'], 'persistent_infos': [b['pd']],
                   'onetime_infos': None})
    _ckpt_roundtrip(tmp_path, lc, ec, sc, bs + [bs[0]])


def test_reference_written_pixel_rnn_checkpoint_restores(tmp_path, golden):
    from surreal_b200.learner import PPOLearner
    g = golden('ppo_learner_ckpt_pixel_rnn')
    cfg = g.js('cfg')
    ck = tmp_path / 'ref' / 'checkpoint'
    ck.mkdir(parents=True)
    names = g.js('file_names') if g['file_names'].ndim == 0 else [str(x) for x in g['file_names']]
    for fn in names:
        (ck / fn).write_bytes(bytes(g['file/' + fn]))
    lc, ec, sc = _gcfg(dict(cfg, mode='clip'))
    sc.folder = str(tmp_path / 'mine')
    sc.checkpoint.restore = True
    sc.checkpoint.restore_folder = str(tmp_path / 'ref')
    L = PPOLearner(lc, ec, sc)
    assert L.current_iteration == cfg['current_iteration']
    for name, model in (('saved/model/', L.model), ('saved/ref/', L.ref_target_model)):
        exp = ref_state_dict(g.sub(name))
        assert 'cnn_stem.model.seq.5.weight' in exp and 'rnn_stem.weight_hh_l0' in exp
        got = model.state_dict()
        assert set(exp) == set(got)
        for k, e in exp.items():
            assert torch.equal(got[k].cpu().reshape(e.shape), e), k


@pytest.mark.parametrize('host', [False, True])
def test_default_config_pixel_rnn_end_to_end(host):
    """PPO_DEFAULT_LEARNER_CONFIG (recurrent, LSTM(100), cnn_feature_dim 256) with use_z_filter off on a [4, 84, 84] pixel
    env, wired by the launcher: the agent's main loop writes windows into the FIFO, the learner's main_loop() trains on
    them for three iterations with finite statistics.  The device run takes the env the agent builds from env_config."""
    import copy
    import tempfile
    from surreal_b200.session import Config
    from surreal_b200.main.ppo_configs import (PPO_DEFAULT_LEARNER_CONFIG, PPO_DEFAULT_ENV_CONFIG, PPO_DEFAULT_SESSION_CONFIG,
                                               make_synthetic_pixel_env_config)
    from surreal_b200.agent import PPOAgent
    from surreal_b200.env import SyntheticPixelEnv
    from surreal_b200.learner import PPOLearner
    from surreal_b200.launch import SurrealDefaultLauncher
    from surreal_b200.replay import FIFOReplay
    lc = Config(copy.deepcopy(PPO_DEFAULT_LEARNER_CONFIG.to_dict()))
    ec = Config(copy.deepcopy(PPO_DEFAULT_ENV_CONFIG.to_dict()))
    sc = Config(copy.deepcopy(PPO_DEFAULT_SESSION_CONFIG.to_dict()))
    sc.folder = tempfile.mkdtemp()
    lc.algo.use_z_filter = False
    N = 64
    make_synthetic_pixel_env_config(ec, N, frame_shape=(4, 84, 84), action_dim=6)
    assert lc.algo.rnn.if_rnn_policy
    la = SurrealDefaultLauncher(PPOAgent, PPOLearner, FIFOReplay, sc, ec, lc)
    env = _HostPixelEnv(SyntheticPixelEnv(N, (4, 84, 84), 6, limit_episode_length=40, seed=1)) if host else None
    agent, replay, learner = la.setup_engine(env=env)
    assert agent.env.host_env == host and agent.env.cells is not None
    stats, real_learn = [], learner.learn

    def learn(batch):
        assert batch['onetime_infos'] is not None and batch['obs']['pixel']['camera0'].dtype == torch.uint8
        stats.append(real_learn(batch))
        return stats[-1]
    learner.learn = learn
    for _ in range(40):
        agent.main_loop(max_steps=lc.algo.stride)
        while replay.start_sample_condition() and len(stats) < 3:
            learner.main_loop()
        if len(stats) >= 3:
            break
    torch.cuda.synchronize()
    assert len(stats) == 3
    for st in stats:
        assert all(np.isfinite(v) for v in st.values()), st


# ---- joint [head | CNN | LSTM] gradients of one policy and one value step against float64 autograd ----------------
GRAD_BAR = 5e-5       # head and LSTM tensors, relative L2 and max error / max|g64| (test_rnn_grads_gpu.py's bar)
CONV_W_BAR, CONV_B_BAR = 5e-5, 1e-4   # CNN stem tensors, max error / max(1, max|g64|) (test_stem_gpu.py's bars)

GRAD_CASES = {                         # C, HW (conv2 output), B, n_step, horizon (eff_len = n - horizon + 1), layers
    'l1_1x1': dict(HW=20, B=8, n=5, horizon=3, layers=1),
    'l2_2x2': dict(HW=28, B=4, n=6, horizon=2, layers=2),
    'l1_3x3_eff1': dict(HW=36, B=16, n=4, horizon=4, layers=1),
    'l2_1x1_long': dict(HW=20, B=32, n=8, horizon=2, layers=2),
}


def _flat_to_torch(stem, buf):
    """A stem's state_items() for the flat buffer ``buf`` (parameters or a gradient) instead of its parameters."""
    keep = stem.params.clone()
    stem.params.copy_(buf)
    items = {k: v.detach().clone() for k, v in stem.state_items()}
    stem.params.copy_(keep)
    return items


def _f64_loss(kind, L, snap, frames, h0, c0, E, actions=None, behave=None):
    """float64 frames -> Conv2d x2 -> Linear + ReLU -> nn.LSTM(num_layers) from (h0, c0) -> head -> the policy (clip) or
    value loss of the learner's rows b*E + t.  -> {name: gradient} in the reference's state_dict names."""
    m = L.model
    head = m.actor if kind == 'policy' else m.critic
    cnn = {k: v.double().cpu().requires_grad_(True) for k, v in _flat_to_torch(m.cnn_stem, snap['cnn']).items()}
    rnn = {k: v.double().cpu().requires_grad_(True) for k, v in _flat_to_torch(m.rnn_stem, snap['rnn']).items()}
    layers = [tuple(t.double().cpu().requires_grad_(True) for t in head.get_layer(l, buf=snap['head'])) for l in range(head.n_layers)]
    B = frames.shape[0]
    p = 'cnn_stem.model.seq.'
    x = torch.as_tensor(frames[:, :E]).reshape(B * E, *frames.shape[2:]).double() / 255.0
    x = torch.relu(F.conv2d(x, cnn[p + '0.weight'], cnn[p + '0.bias'], stride=4))
    x = torch.relu(F.conv2d(x, cnn[p + '2.weight'], cnn[p + '2.bias'], stride=2)).flatten(1)
    x = torch.relu(F.linear(x, cnn[p + '5.weight'], cnn[p + '5.bias']))
    nl, Hd = m.rnn_stem.layers, m.rnn_stem.H
    lstm = torch.nn.LSTM(x.shape[1], Hd, nl, batch_first=True).double()
    out, _ = torch.func.functional_call(lstm, {k[len('rnn_stem.'):]: v for k, v in rnn.items()},
                                        (x.view(B, E, -1), (torch.as_tensor(h0).double().transpose(0, 1).contiguous(),
                                                            torch.as_tensor(c0).double().transpose(0, 1).contiguous())))
    h = out.reshape(B * E, Hd)
    for l, (w, b) in enumerate(layers):
        h = F.linear(h, w, b)
        if l < len(layers) - 1:
            h = torch.relu(h)
    leaves = dict(cnn, **rnn)
    for l, (w, b) in enumerate(layers):
        leaves['head.%d.weight' % l], leaves['head.%d.bias' % l] = w, b
    if kind == 'policy':
        import grad_ref as R
        A = L.action_dim
        lv = head.extra_view(snap['head']).double().cpu().requires_grad_(True)
        leaves['log_var'] = lv
        loss, _ = R._policy_loss(h, lv, torch.as_tensor(actions[:, :E]).double().reshape(-1, A), L._adv.double().cpu().reshape(-1),
                                 torch.as_tensor(behave[:, :E]).double().reshape(-1, 2 * A), 'clip', clip_eps=L.clip_epsilon)
    else:
        loss = (h - L._ret.double().cpu().reshape(-1, 1)).pow(2).mean()
    gs = torch.autograd.grad(loss, list(leaves.values()))
    return dict(zip(leaves, gs))


def _check_grad(L, kind, g, ref):
    m = L.model
    head = m.actor if kind == 'policy' else m.critic
    nh, nc = head.size, m.cnn_stem.size
    got = dict(_flat_to_torch(m.cnn_stem, g[nh:nh + nc]), **_flat_to_torch(m.rnn_stem, g[nh + nc:]))
    for l in range(head.n_layers):
        got['head.%d.weight' % l], got['head.%d.bias' % l] = head.get_layer(l, buf=g[:nh])
    if kind == 'policy':
        got['log_var'] = head.extra_view(g[:nh])
    worst = {}
    for k, e in ref.items():
        d = got[k].double().cpu().reshape(e.shape)
        err = float((d - e).abs().max())
        if k.startswith('cnn_stem.'):
            r = err / max(1.0, float(e.abs().max()))
            assert r <= (CONV_W_BAR if k.endswith('weight') else CONV_B_BAR), (kind, k, r)
        else:
            r = max(float((d - e).norm()) / max(float(e.norm()), 1e-30), err / max(float(e.abs().max()), 1e-30))
            assert r <= GRAD_BAR, (kind, k, r)
        worst[k] = r
    print('measured', kind, max(worst.values()))


@pytest.mark.parametrize('case', list(GRAD_CASES))
def test_pixel_rnn_joint_gradients_match_float64(case, monkeypatch):
    """One policy epoch and one value epoch of eager learn(): the [head | CNN | LSTM] gradient each optimiser steps matches
    float64 autograd (Conv2d x2, Linear, nn.LSTM(num_layers), heads) at the parameters that epoch starts from -- the value
    epoch on the stems the policy step has already moved."""
    from surreal_b200.learner import PPOLearner
    c = GRAD_CASES[case]
    monkeypatch.setenv('SB200_CUDA_GRAPH', '0')
    C, A, Hd, Fd = 2, 3, 10, 12
    lc, ec, sc = _cfg(C, c['HW'], Fd, A, [32, 24], [28, 20], c['n'], c['B'], 'clip', 1e-3, 10 ** 6, c['horizon'], Hd,
                      c['layers'])
    lc.algo.consts.epoch_policy = lc.algo.consts.epoch_baseline = 1
    torch.manual_seed(11)
    L = PPOLearner(lc, ec, sc)
    L.use_cuda_graph = False
    B, n, E, nl = c['B'], c['n'], L.eff_len, c['layers']
    rng = np.random.default_rng(7)
    obs = rng.integers(0, 256, size=(B, n, C, c['HW'], c['HW']), dtype=np.uint8)
    obs_next = rng.integers(0, 256, size=(B, 1, C, c['HW'], c['HW']), dtype=np.uint8)
    h0 = (rng.standard_normal((B, nl, Hd)) * 0.3).astype(np.float32)
    c0 = (rng.standard_normal((B, nl, Hd)) * 0.5).astype(np.float32)
    mean = np.tanh(rng.standard_normal((B, n, A)) * 0.5).astype(np.float32)
    std = np.exp(rng.uniform(-1.2, -0.6, size=(B, 1, A))).astype(np.float32).repeat(n, 1)
    pd = np.concatenate([mean, std], 2)
    actions = np.clip(mean + std * rng.standard_normal((B, n, A)), -1, 1).astype(np.float32)
    batch = {'obs': {'pixel': {'camera0': obs}}, 'obs_next': {'pixel': {'camera0': obs_next}}, 'actions': actions,
             'rewards': (rng.standard_normal((B, n)) * 0.5).astype(np.float32), 'dones': (rng.random((B, n)) < 0.1).astype(np.float32),
             'persistent_infos': [pd], 'onetime_infos': [h0, c0]}
    rec = {}
    m = L.model
    for kind, fn, head, g in (('policy', '_policy_epoch', m.actor, '_g_actor'), ('value', '_value_epoch', m.critic, '_g_critic')):
        orig = getattr(L, fn)

        def wrapped(*a, _orig=orig, _kind=kind, _head=head, _g=g, **k):
            snap = {'head': _head.params.clone(), 'cnn': m.cnn_stem.params.clone(), 'rnn': m.rnn_stem.params.clone()}
            _orig(*a, **k)
            rec[_kind] = (snap, getattr(L, _g).clone())
        setattr(L, fn, wrapped)
    L.learn(batch)
    torch.cuda.synchronize()
    assert not torch.equal(rec['value'][0]['cnn'], rec['policy'][0]['cnn'])      # the value step sees the stepped stems
    for kind in ('policy', 'value'):
        snap, g = rec[kind]
        ref = _f64_loss(kind, L, snap, obs, h0, c0, E, actions=actions, behave=pd)
        _check_grad(L, kind, g, ref)

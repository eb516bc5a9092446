#!/usr/bin/env python
"""Generate the golden vectors of the CNN + LSTM policy (pixel input with algo.rnn.if_rnn_policy, the reference's default
PPO config on a camera env) by running the REAL reference, with the harness and helpers of make_golden.py (run in the
build container only, like it):

    python tests/golden/make_golden_pixel_rnn.py          # writes the fixtures below

  fixture                          reference code that produced it
  -------------------------------  ----------------------------------------------------------------------------------
  ppo_learn_pixel_rnn_clip.npz     surreal/learner/ppo.py:420-666 with uint8 frame -> CNN stem -> nn.LSTM -> heads
                                   (ppo_net.py:136-156,268-279; builders.py:23-33 for the 5-D [B, T, C, H, W] frames)
  ppo_learn_pixel_rnn_adapt.npz    the same in adapt mode, learning rate high enough for the KL early stop (ppo.py:556)
  ppo_learn_pixel_rnn2_clip.npz    the same with rnn_layer = 2 and 28x28 frames (conv2 output 2x2)
  ppo_act_pixel_rnn.npz            surreal/agent/ppo_agent.py:84-93,133-137,169-183 on frames, cells handed off, reset
  ppo_learner_ckpt_pixel_rnn.npz   surreal/utils/checkpoint.py:18-347 files of a pixel + LSTM PPOLearner

Frames are uint8 [C, H, W]; the cells of a window's first step travel as onetime_infos [B, rnn_layer, H]."""
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (installs the reference harness)

import numpy as np  # noqa: E402
import torch  # noqa: E402

H = G.H
PPOLearner, PPOAgent, save, sd_np = G.PPOLearner, G.PPOAgent, G.save, G.sd_np
C, F = 2, 12


def cfg_pixel_rnn(HW, rnn_layer=1, **kw):
    lc, ec, sc = G.cfg_ppo(rnn=True, use_z=False, **kw)
    ec.obs_spec = {'pixel': {'camera0': (C, HW, HW)}}
    ec.pixel_input = True
    lc.model.cnn_feature_dim = F
    lc.algo.rnn.rnn_layer = rnn_layer
    return lc, ec, sc


def make_batch(L, rng, HW):
    """Random frames, the behaviour policy from the reference model itself (zero cells), scaled exploration noise."""
    B, n, A = L.batch_size, L.n_step, L.action_dim
    Hd, Lr = L.learner_config.algo.rnn.rnn_hidden, L.learner_config.algo.rnn.rnn_layer
    obs = rng.integers(0, 256, size=(B, n, C, HW, HW), dtype=np.uint8)
    obs_next = rng.integers(0, 256, size=(B, 1, C, HW, HW), dtype=np.uint8)
    with torch.no_grad():
        h0 = torch.zeros(Lr, B, Hd)
        pd = L.model.forward_actor({'pixel': {'camera0': torch.tensor(obs, dtype=torch.float32)}}, (h0, h0.clone()))
        pd = pd.numpy().reshape(B, n, 2 * A).copy()
    pd[:, :, A:] *= np.exp(rng.uniform(-0.25, 0.25, size=(B, 1, 1))).astype(np.float32)
    actions = np.clip(rng.standard_normal((B, n, A)) * pd[:, :, A:] + pd[:, :, :A], -1, 1)
    rewards = rng.standard_normal((B, n)) * 0.5 + 0.1
    dones = np.zeros((B, n), dtype=np.float32)
    dones[rng.random(B) < 0.3, n - 1] = 1.0
    h = (rng.standard_normal((B, Lr, Hd)) * 0.1).astype(np.float32)
    c = (rng.standard_normal((B, Lr, Hd)) * 0.1).astype(np.float32)
    batch = H._AttrDict(obs={'pixel': {'camera0': obs.copy()}}, obs_next={'pixel': {'camera0': obs_next.copy()}},
                        actions=actions.copy(), rewards=rewards.copy(), dones=dones.copy(),
                        persistent_infos=[pd.astype(np.float32).copy()], onetime_infos=[h.copy(), c.copy()])
    raw = dict(obs=obs, obs_next=obs_next, actions=actions, rewards=rewards, dones=dones, pd=pd.astype(np.float32),
               h0=h, c0=c)
    return batch, raw


def gen_ppo_learn_pixel_rnn():
    """learn() + publish for two iterations: the CNN and the LSTM stem trained by BOTH optimisers (ppo_net.py:202-224)."""
    variants = [
        ('pixel_rnn_clip', 20, 1, dict(mode='clip', B=6, n_step=5, stride=5, horizon=3, rnn_hidden=6, exp_interval=12)),
        ('pixel_rnn_adapt', 20, 1, dict(mode='adapt', B=6, n_step=5, stride=5, horizon=2, rnn_hidden=6, lr=5e-3,
                                        exp_interval=12)),
        ('pixel_rnn2_clip', 28, 2, dict(mode='clip', B=4, n_step=5, stride=5, horizon=3, rnn_hidden=7, exp_interval=8)),
    ]
    for tag, HW, layers, kw in variants:
        torch.manual_seed(29)
        lc, ec, sc = cfg_pixel_rnn(HW, layers, **kw)
        L = H.construct_without_initialize(PPOLearner, lc, ec, sc)
        L._ps_publisher = H._Any()
        L.tensorplex = H._Any()
        L.ref_target_model.update_target_params(L.model)
        rng = np.random.default_rng(29)
        out = dict(**sd_np(L.model, 'init/'))
        n_pol = []
        name = '_clip_update' if L.ppo_mode == 'clip' else '_adapt_update'
        orig_update = getattr(L, name)

        def counting(*a, **k):
            n_pol[-1] += 1
            return orig_update(*a, **k)
        setattr(L, name, counting)
        stats_all, hyper, captured = [], [], {}
        orig_opt, orig_gae = L._optimize, L._gae_and_return

        def opt_hook(*a, **k):
            st = orig_opt(*a, **k)
            captured['stats'] = {kk: float(vv) for kk, vv in st.items()}
            return st

        def gae_hook(*a, **k):
            adv, ret = orig_gae(*a, **k)
            captured['adv'], captured['ret'] = adv.detach().clone().numpy(), ret.detach().clone().numpy()
            return adv, ret
        L._optimize, L._gae_and_return = opt_hook, gae_hook
        for it in range(2):
            batch, raw = make_batch(L, rng, HW)
            for k, v in raw.items():
                out['it%d/%s' % (it, k)] = v
            n_pol.append(0)
            L.learn(batch)
            stats_all.append(captured['stats'])
            out['it%d/adv' % it], out['it%d/ret' % it] = captured['adv'], captured['ret']
            L.publish_parameter(it, message='')
            out.update(sd_np(L.model, 'it%d/after/' % it))
            hyper.append(dict(clip_epsilon=getattr(L, 'clip_epsilon', None), beta=getattr(L, 'beta', None),
                              exp_counter=L.exp_counter, n_policy_epochs=n_pol[-1],
                              kl_record=list(map(float, L.kl_record))))
        print(tag, 'policy epochs per iteration:', n_pol)
        cfg = dict(mode=L.ppo_mode, B=L.batch_size, n_step=L.n_step, A=L.action_dim, C=C, HW=HW, cnn_feature_dim=F,
                   actor_h=lc.model.actor_fc_hidden_sizes, critic_h=lc.model.critic_fc_hidden_sizes,
                   lr=lc.algo.network.lr_actor, exp_interval=lc.parameter_publish.exp_interval, iters=2,
                   horizon=L.horizon, rnn_hidden=lc.algo.rnn.rnn_hidden, rnn_layer=layers,
                   epoch_policy=L.epoch_policy, epoch_baseline=L.epoch_baseline)
        save('ppo_learn_' + tag, cfg=cfg, stats=stats_all, hyper=hyper, **out)


def gen_act_pixel_rnn():
    """PPOAgent.act on single uint8 frames with the CNN + LSTM model: the cells BEFORE each step are its onetime_infos,
    reset() zeroes them."""
    HW = 20
    torch.manual_seed(47)
    lc, ec, sc = cfg_pixel_rnn(HW, 1, A=3, horizon=3, rnn_hidden=6)
    sc.agent.num_gpus = 0
    np.random.seed(47)
    Ag = H.construct_without_initialize(PPOAgent, lc, ec, sc, 2, 'training')
    noise = Ag.noise
    rng = np.random.default_rng(47)
    obs = rng.integers(0, 256, size=(7, C, HW, HW), dtype=np.uint8)
    np.random.seed(4747)
    eps = np.random.randn(7, 1, 3)
    np.random.seed(4747)
    acts, pds, h_before, c_before = [], [], [], []
    for i in range(7):
        if i == 4:
            Ag.reset()
        a, info = Ag.act({'pixel': {'camera0': obs[i]}})
        acts.append(a)
        pds.append(info[1][0])
        h_before.append(info[0][0])
        c_before.append(info[0][1])
    save('ppo_act_pixel_rnn', obs=obs, eps=eps[:, 0, :], noise=noise, actions=np.stack(acts), pds=np.stack(pds),
         h_before=np.stack(h_before), c_before=np.stack(c_before), reset_at=4, rnn_hidden=6, C=C, HW=HW,
         cnn_feature_dim=F, **sd_np(Ag.model, 'model/'))


def gen_ppo_learner_ckpt_pixel_rnn():
    """A checkpoint folder written by the REFERENCE for a pixel + LSTM PPOLearner (state_dict keys cnn_stem.model.seq.*
    and rnn_stem.*_l0), after two learn() + publish iterations, with the state it holds."""
    from surreal.utils.checkpoint import PeriodicCheckpoint
    HW = 20
    torch.manual_seed(31)
    lc, ec, sc = cfg_pixel_rnn(HW, 1, mode='clip', B=4, n_step=5, stride=5, horizon=3, rnn_hidden=6, exp_interval=8)
    L = H.construct_without_initialize(PPOLearner, lc, ec, sc)
    L._ps_publisher = H._Any()
    L.tensorplex = H._Any()
    L.ref_target_model.update_target_params(L.model)
    rng = np.random.default_rng(31)
    folder = tempfile.mkdtemp()
    ck = PeriodicCheckpoint(folder, 'learner', period=1, min_interval=0, tracked_obj=L,
                            tracked_attrs=L.checkpoint_attributes(), keep_history=2, keep_best=0)
    L.periodic_checkpoint = lambda **kw_: None
    for it in range(2):
        batch, _ = make_batch(L, rng, HW)
        L.learn(batch)
        L.publish_parameter(it, message='')
    ck.save(score=None, global_steps=L.current_iteration)
    out = dict(**sd_np(L.model, 'saved/model/'), **sd_np(L.ref_target_model, 'saved/ref/'))
    files = {fn: np.frombuffer(open(os.path.join(folder, fn), 'rb').read(), dtype=np.uint8) for fn in sorted(os.listdir(folder))}
    save('ppo_learner_ckpt_pixel_rnn', file_names=sorted(files),
         cfg=dict(B=L.batch_size, n_step=L.n_step, A=L.action_dim, C=C, HW=HW, cnn_feature_dim=F, exp_interval=8,
                  horizon=3, rnn_hidden=6, rnn_layer=1, actor_h=lc.model.actor_fc_hidden_sizes,
                  critic_h=lc.model.critic_fc_hidden_sizes, lr=lc.algo.network.lr_actor,
                  current_iteration=int(L.current_iteration)),
         **{'file/' + k: v for k, v in files.items()}, **out)


if __name__ == '__main__':
    which = sys.argv[1:] or ['ppo_learn_pixel_rnn', 'act_pixel_rnn', 'ppo_learner_ckpt_pixel_rnn']
    for w in which:
        globals()['gen_' + w]()

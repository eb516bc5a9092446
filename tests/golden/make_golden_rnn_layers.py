#!/usr/bin/env python
"""Generate the golden vectors of stacked LSTM stems (algo.rnn.rnn_layer > 1) by running the REAL reference, with the
harness and helpers of make_golden.py (run in the build container only, like it):

    python tests/golden/make_golden_rnn_layers.py          # writes the fixtures below

  fixture                       reference code that produced it
  ----------------------------  -------------------------------------------------------------------------------------
  ppo_learn_rnn2_clip.npz       surreal/learner/ppo.py:420-666 with nn.LSTM(.., rnn_layer=2) (ppo_net.py:143-152)
  ppo_learn_rnn2_adapt.npz      the same in adapt mode, learning rate high enough for the KL early stop (ppo.py:556)
  ppo_learn_rnn3_clip.npz       the same with rnn_layer = 3
  ppo_act_rnn2.npz              surreal/agent/ppo_agent.py:84-93,133-137,169-183 with cells (2, 1, H)
  ppo_learner_ckpt_rnn2.npz     surreal/utils/checkpoint.py:18-347 files of a PPOLearner with a 2-layer LSTM

The initial cells are [rnn_layer, B, H] for the behaviour-policy forward and travel as onetime_infos [B, rnn_layer, H]
(ppo_agent.py:133-135, learner/ppo.py:507-510)."""
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (installs the reference harness)

import numpy as np  # noqa: E402
import torch  # noqa: E402

H = G.H
PPOLearner, PPOAgent, save, sd_np = G.PPOLearner, G.PPOAgent, G.save, G.sd_np


def cfg_ppo(rnn_layer, **kw):
    lc, ec, sc = G.cfg_ppo(**kw)
    lc.algo.rnn.rnn_layer = rnn_layer
    return lc, ec, sc


def make_ppo_batch(L, rng, B, n, D, A, log_sig_range=0.25, done_last_frac=0.25):
    """make_golden.make_ppo_batch with [rnn_layer, B, H] initial cells for the pd forward and [B, rnn_layer, H]
    onetime_infos (RNN mode only)."""
    Hd, Lr = L.learner_config.algo.rnn.rnn_hidden, L.learner_config.algo.rnn.rnn_layer
    obs = rng.standard_normal((B, n, D)).astype(np.float32) * 1.5 + 0.3
    obs_next = rng.standard_normal((B, 1, D)).astype(np.float32) * 1.5 + 0.3
    with torch.no_grad():
        flat = {'low_dim': {'flat_inputs': torch.tensor(obs)}}
        h0 = torch.zeros(Lr, B, Hd)
        pd = L.model.forward_actor(flat, (h0, h0.clone())).numpy().reshape(B, n, 2 * A)
    noise = rng.uniform(-log_sig_range, log_sig_range, size=(B, 1, 1))
    pd = pd.copy()
    pd[:, :, A:] *= np.exp(noise).astype(np.float32)           # ppo_agent.py:139
    eps = rng.standard_normal((B, n, A))
    actions = np.clip(eps * pd[:, :, A:] + pd[:, :, :A], -1, 1)
    rewards = rng.standard_normal((B, n)) * 0.5 + 0.1
    dones = np.zeros((B, n), dtype=np.float32)
    dones[rng.random(B) < done_last_frac, n - 1] = 1.0
    h = (rng.standard_normal((B, Lr, Hd)) * 0.1).astype(np.float32)
    c = (rng.standard_normal((B, Lr, Hd)) * 0.1).astype(np.float32)
    batch = H._AttrDict(
        obs={'low_dim': {'flat_inputs': obs.copy()}},
        obs_next={'low_dim': {'flat_inputs': obs_next.copy()}},
        actions=actions.copy(), rewards=rewards.copy(), dones=dones.copy(),
        persistent_infos=[pd.astype(np.float32).copy()], onetime_infos=[h.copy(), c.copy()])
    raw = dict(obs=obs, obs_next=obs_next, actions=actions, rewards=rewards, dones=dones, pd=pd.astype(np.float32),
               h0=h, c0=c)
    return batch, raw


def gen_ppo_learn_rnn_layers():
    """learn() + publish for a few iterations, every layer of the LSTM trained by BOTH optimisers (ppo_net.py:202-224)."""
    variants = [
        ('rnn2_clip', 2, dict(mode='clip', B=8, n_step=7, rnn=True, horizon=3, rnn_hidden=10, exp_interval=16), 3),
        ('rnn2_adapt', 2, dict(mode='adapt', B=8, n_step=6, rnn=True, horizon=2, rnn_hidden=6, lr=2e-2, exp_interval=8), 2),
        ('rnn3_clip', 3, dict(mode='clip', B=6, n_step=5, rnn=True, horizon=2, rnn_hidden=7, exp_interval=12), 2),
    ]
    for tag, layers, kw, iters in variants:
        torch.manual_seed(13)
        lc, ec, sc = cfg_ppo(layers, **kw)
        L = H.construct_without_initialize(PPOLearner, lc, ec, sc)
        L._ps_publisher = H._Any()
        L.tensorplex = H._Any()
        rng = np.random.default_rng(13)
        B, n, D, A = L.batch_size, L.n_step, 11, 3
        L.model.z_filter.z_update(torch.tensor((rng.standard_normal((40, D)) * 1.5 + 0.3).astype(np.float32)))
        L.ref_target_model.update_target_params(L.model)
        out = dict(**sd_np(L.model, 'init/'))
        n_pol = []
        orig_update = L._clip_update if L.ppo_mode == 'clip' else L._adapt_update

        def counting(*a, **k):
            n_pol[-1] += 1
            return orig_update(*a, **k)
        if L.ppo_mode == 'clip':
            L._clip_update = counting
        else:
            L._adapt_update = counting
        stats_all, hyper = [], []
        captured = {}
        orig_opt = L._optimize
        orig_gae = L._gae_and_return

        def opt_hook(*a, **k):
            st = orig_opt(*a, **k)
            captured['stats'] = {kk: float(vv) for kk, vv in st.items()}
            return st

        def gae_hook(*a, **k):
            adv, ret = orig_gae(*a, **k)
            captured['adv'], captured['ret'] = adv.detach().clone().numpy(), ret.detach().clone().numpy()
            return adv, ret
        L._optimize = opt_hook
        L._gae_and_return = gae_hook
        for it in range(iters):
            batch, raw = make_ppo_batch(L, rng, B, n, D, A)
            for k, v in raw.items():
                out['it%d/%s' % (it, k)] = v
            n_pol.append(0)
            L.learn(batch)
            stats_all.append(captured['stats'])
            out['it%d/adv' % it], out['it%d/ret' % it] = captured['adv'], captured['ret']
            L.publish_parameter(it, message='')
            out.update(sd_np(L.model, 'it%d/after/' % it))
            out.update(sd_np(L.ref_target_model, 'it%d/ref/' % it))
            hyper.append(dict(clip_epsilon=getattr(L, 'clip_epsilon', None), beta=getattr(L, 'beta', None),
                              exp_counter=L.exp_counter, n_policy_epochs=n_pol[-1],
                              kl_record=list(map(float, L.kl_record))))
        cfg = dict(mode=L.ppo_mode, B=B, n_step=n, D=D, A=A, actor_h=lc.model.actor_fc_hidden_sizes,
                   critic_h=lc.model.critic_fc_hidden_sizes, lr=lc.algo.network.lr_actor, gamma=L.gamma,
                   lam=L.lam, exp_interval=lc.parameter_publish.exp_interval, iters=iters, horizon=L.horizon,
                   rnn_hidden=lc.algo.rnn.rnn_hidden, rnn_layer=lc.algo.rnn.rnn_layer,
                   kl_target=L.kl_target, epoch_policy=L.epoch_policy, epoch_baseline=L.epoch_baseline)
        save('ppo_learn_' + tag, cfg=cfg, stats=stats_all, hyper=hyper, **out)


def gen_act_rnn2():
    """PPOAgent.act with a 2-layer LSTM: cells (2, 1, H) carried by the agent, the cells BEFORE each step are the
    onetime_infos (2, H) of that step, reset() zeroes them."""
    torch.manual_seed(43)
    lc, ec, sc = cfg_ppo(2, D=11, A=3, rnn=True, horizon=3, rnn_hidden=10)
    sc.agent.num_gpus = 0
    np.random.seed(43)
    Ag = H.construct_without_initialize(PPOAgent, lc, ec, sc, 2, 'training')
    noise = Ag.noise
    rng = np.random.default_rng(43)
    Ag.model.z_filter.z_update(torch.tensor((rng.standard_normal((40, 11)) * 1.5 + 0.3).astype(np.float32)))
    obs = rng.standard_normal((7, 11)).astype(np.float32)
    np.random.seed(4343)
    eps = np.random.randn(7, 1, 3)
    np.random.seed(4343)
    acts, pds, h_before, c_before = [], [], [], []
    for i in range(7):
        if i == 4:
            Ag.reset()
        a, info = Ag.act({'low_dim': {'flat_inputs': obs[i]}})
        acts.append(a)
        pds.append(info[1][0])
        h_before.append(info[0][0])
        c_before.append(info[0][1])
    save('ppo_act_rnn2', obs=obs, eps=eps[:, 0, :], noise=noise, actions=np.stack(acts), pds=np.stack(pds),
         h_before=np.stack(h_before), c_before=np.stack(c_before), reset_at=4, rnn_hidden=10,
         **sd_np(Ag.model, 'model/'))


def gen_ppo_learner_ckpt_rnn2():
    """A checkpoint folder written by the REFERENCE for an RNN-mode PPOLearner with a 2-layer LSTM (state_dict keys
    rnn_stem.{weight,bias}_{ih,hh}_l{0,1}), after two learn() + publish iterations, with the state it holds."""
    from surreal.utils.checkpoint import PeriodicCheckpoint
    torch.manual_seed(23)
    lc, ec, sc = cfg_ppo(2, mode='clip', B=8, n_step=6, rnn=True, horizon=2, rnn_hidden=9, exp_interval=8)
    L = H.construct_without_initialize(PPOLearner, lc, ec, sc)
    L._ps_publisher = H._Any()
    L.tensorplex = H._Any()
    rng = np.random.default_rng(23)
    B, n, D, A = L.batch_size, L.n_step, 11, 3
    L.model.z_filter.z_update(torch.tensor((rng.standard_normal((40, D)) * 1.5 + 0.3).astype(np.float32)))
    L.ref_target_model.update_target_params(L.model)
    folder = tempfile.mkdtemp()
    ck = PeriodicCheckpoint(folder, 'learner', period=1, min_interval=0, tracked_obj=L,
                            tracked_attrs=L.checkpoint_attributes(), keep_history=2, keep_best=0)
    L.periodic_checkpoint = lambda **kw_: None
    for it in range(2):
        batch, raw = make_ppo_batch(L, rng, B, n, D, A)
        L.learn(batch)
        L.publish_parameter(it, message='')
    ck.save(score=None, global_steps=L.current_iteration)
    out = dict(**sd_np(L.model, 'saved/model/'), **sd_np(L.ref_target_model, 'saved/ref/'))
    files = {fn: np.frombuffer(open(os.path.join(folder, fn), 'rb').read(), dtype=np.uint8) for fn in sorted(os.listdir(folder))}
    save('ppo_learner_ckpt_rnn2', file_names=sorted(files), cfg=dict(B=B, n_step=n, D=D, A=A, exp_interval=8, horizon=2,
         rnn_hidden=9, rnn_layer=2, actor_h=lc.model.actor_fc_hidden_sizes, critic_h=lc.model.critic_fc_hidden_sizes,
         lr=lc.algo.network.lr_actor, current_iteration=int(L.current_iteration)),
         **{'file/' + k: v for k, v in files.items()}, **out)


if __name__ == '__main__':
    which = sys.argv[1:] or ['ppo_learn_rnn_layers', 'act_rnn2', 'ppo_learner_ckpt_rnn2']
    for w in which:
        globals()['gen_' + w]()

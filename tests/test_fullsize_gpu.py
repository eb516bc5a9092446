"""Full BASELINE-size cases (configs[1], [2], [4]) on the GPU: one learn() against the CPU oracle on identical
seeded inputs, plus size-independent properties (index-stream identity, gather checksums, FIFO conservation)."""
import random

import numpy as np
import pytest
import torch

from helpers import ppo_configs, ddpg_configs
from oracle import nets as onets
from oracle.filters import ZFilter as OZ
from oracle.ppo import OraclePPOLearner
from oracle.ddpg import OracleDDPGLearner

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _layers(dims, gen, aux=0, aux_layer=-1):
    out = []
    for i in range(len(dims) - 1):
        k = dims[i] + (aux if aux_layer == i else 0)
        b = 1.0 / np.sqrt(k)
        out.append(((torch.rand(dims[i + 1], k, generator=gen) * 2 - 1) * b, (torch.rand(dims[i + 1], generator=gen) * 2 - 1) * b))
    return out


@pytest.mark.parametrize('B,n,mode', [(1024, 128, 'clip'), (1024, 128, 'adapt'), (4096, 64, 'clip')])
def test_ppo_learn_fullsize_vs_oracle(B, n, mode):
    """configs[1] (1024 x 128, 64-dim obs, A = 8, 2x256 MLP) and a 4096-window batch: losses, KL, advantages
    and updated parameters against the oracle (torch-CPU autograd + torch.optim.Adam)."""
    from surreal_b200.learner import PPOLearner
    D, A = 64, 8
    gen = torch.Generator().manual_seed(B + n)
    al, cl = _layers([D, 256, 256, A], gen), _layers([D, 256, 256, 1], gen)
    log_var = torch.zeros(1, A) - 1.0
    zf = OZ(D)
    zf.update(torch.randn(500, D, generator=gen) * 1.3 + 0.2)
    rng = np.random.default_rng(B)
    obs = (rng.standard_normal((B, n, D)) * 1.2).astype(np.float32)
    obs_next = (rng.standard_normal((B, 1, D)) * 1.2).astype(np.float32)
    with torch.no_grad():
        pd0 = onets.ppo_actor(zf.forward(torch.tensor(obs[:, 0])), al, log_var).numpy()
    pd = np.tile(pd0[:, None, :], (1, n, 1)).astype(np.float32)
    pd[:, :, A:] *= np.exp(rng.uniform(-0.25, 0.25, (B, 1, 1))).astype(np.float32)
    actions = np.clip(rng.standard_normal((B, n, A)) * pd[:, :, A:] + pd[:, :, :A], -1, 1)
    rewards = rng.standard_normal((B, n)) * 0.3
    dones = np.zeros((B, n), dtype=np.float32)
    dones[rng.random(B) < 0.3, n - 1] = 1
    O = OraclePPOLearner(al, log_var, cl, zf, A, n, B, ppo_mode=mode)
    st_o = O.learn(dict(obs=obs, obs_next=obs_next, actions=actions, rewards=rewards, dones=dones, pd=pd))
    lc, ec, sc = ppo_configs(D=D, A=A, actor_h=(256, 256), critic_h=(256, 256), n_step=n, stride=n, B=B, mode=mode)
    L = PPOLearner(lc, ec, sc)
    L.model.actor.load_layers(al, extra=log_var)
    L.model.critic.load_layers(cl)
    # the oracle cloned `zf` at construction, so `zf` still holds the initial statistics
    L.model.z_stats.copy_(torch.cat([zf.running_sum, zf.running_sumsq, zf.count]).to(DEV))
    L.ref_target_model.update_target_params(L.model)
    st = L.learn({'obs': obs, 'obs_next': obs_next, 'actions': actions, 'rewards': rewards, 'dones': dones,
                  'persistent_infos': [pd], 'onetime_infos': None})
    torch.cuda.synchronize()
    assert L.last_n_policy_epochs == O.n_policy_epochs[-1]
    adv, ret = L._adv.cpu().view(-1), L._ret.cpu().view(-1)
    assert float((adv - O.last_adv.view(-1)).abs().max()) <= 1e-5                       # normalised advantages
    rms = float(O.last_ret.pow(2).mean().sqrt())
    assert float((ret - O.last_ret.view(-1)).abs().max()) <= 1e-5 * max(1.0, rms)
    for k in ['_surr_loss', '_clip_surr_loss', '_kl_loss_adapt', '_pol_kl', '_val_loss', '_entropy', '_avg_return_targ',
              '_avg_is_weight', '_ref_behave_diff']:
        if k in st_o:
            assert abs(st[k] - st_o[k]) <= 1e-5 * max(1.0, abs(st_o[k])), (k, st[k], st_o[k])
    # the gradient norms of the last policy / value step: measured worst 2.4e-7 relative; bar 2e-6
    for k in ('grad_norm_actor', 'grad_norm_critic'):
        assert abs(st[k] - st_o[k]) <= 2e-6 * abs(st_o[k]), (k, st[k], st_o[k])
    diffs = []
    for l in range(3):
        for got, exp in ((L.model.actor.get_layer(l), O.actor[l]), (L.model.critic.get_layer(l), O.critic[l])):
            diffs.append((got[0].cpu() - exp[0].detach()).abs().view(-1))
            diffs.append((got[1].cpu() - exp[1].detach()).abs().view(-1))
    diffs.append((L.model.log_var.cpu() - O.log_var.detach().view(-1)).abs().view(-1))
    _assert_params_close(torch.cat(diffs), lr=1e-4, steps=20)
    # The Adam moments, unlike the parameters, scale with the gradient: the oracle's torch.optim.Adam state mapped into
    # kernel layout, per tensor relative L2.  Measured worst 1.9e-4 (4096 x 64, clip); bar 1e-3.
    for net, tr, opt, layers, lv in ((L.model.actor, L.actor_optim, O.actor_optim, O.actor, O.log_var),
                                     (L.model.critic, L.critic_optim, O.critic_optim, O.critic, None)):
        for key, buf in (('exp_avg', tr.exp_avg), ('exp_avg_sq', tr.exp_avg_sq)):
            pairs = []
            for l, (w, b) in enumerate(layers):
                gw, gb = net.get_layer(l, buf=buf)
                pairs += [(gw, opt.state[w][key]), (gb, opt.state[b][key])]
            if lv is not None:
                pairs.append((net.extra_view(buf), opt.state[lv][key].view(-1)))
            for got, exp in pairs:
                e = float((got.cpu().double() - exp.double()).norm()) / max(float(exp.double().norm()), 1e-30)
                assert e <= MOM_BAR, (key, e)


MOM_BAR = 1e-3


def _assert_params_close(d, lr, steps):
    """Parameters after Adam steps.  Adam divides by sqrt(v)+1e-8: for the weights whose gradient is ~0 (|g| < ~1e-8)
    rounding noise alone decides the direction of a full-size step, so the max-abs difference is not a meaningful
    bar.  Robust form: the bulk agrees to a small fraction of ONE step, outliers are rare and bounded by the steps
    taken.  (The parity bar proper -- advantages, returns, losses, KL at 1e-5 -- is asserted above.)"""
    rms = float(d.pow(2).mean().sqrt())
    frac = float((d > 0.05 * lr).float().mean())
    assert float(d.median()) <= 0.002 * lr, ('median', float(d.median()))
    assert rms <= 0.1 * lr, ('rms', rms)
    assert frac <= 0.02, ('fraction beyond 5% of a step', frac)
    assert float(d.max()) <= 2.0 * steps * lr, ('max', float(d.max()))


def test_ddpg_fullsize_uniform_replay_and_learn():
    """configs[2]: 1 048 576-slot UniformReplay in HBM, batch 4096, nets 300-200 / 400-300, gamma^3."""
    from surreal_b200.replay import UniformReplay
    from surreal_b200.learner import DDPGLearner
    D, A, B, CAP = 64, 8, 4096, 1 << 20
    lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=(300, 200), critic_h=(400, 300), B=B, n_step=3, memory_size=CAP, start=3000)
    R = UniformReplay(lc, ec, sc)
    g = torch.Generator(device=DEV).manual_seed(4)
    # pre-fill the ring device-side (SURVEY §8d cfg 3): the k-th record lands in slot k % capacity
    R.r_obs.copy_(torch.randn(CAP, D, device=DEV, generator=g))
    R.r_obs_next.copy_(torch.randn(CAP, D, device=DEV, generator=g))
    R.r_act.copy_(torch.rand(CAP, A, device=DEV, generator=g) * 2 - 1)
    R.r_rew.copy_(torch.randn(CAP, device=DEV, generator=g))
    R.r_done.copy_((torch.rand(CAP, device=DEV, generator=g) < 0.005).float())
    R.state[0], R.state[1] = 0, CAP
    R.mark_device_inserts()
    assert len(R) == CAP and R.start_sample_condition()
    random.seed(5)
    expect = [random.randint(0, CAP - 1) for _ in range(B)]
    random.seed(5)
    batch = R.sample(B)
    idx = batch['indices'].tolist()
    assert idx == expect                                              # bit-exact CPython index stream
    ti = torch.tensor(idx, device=DEV)
    for got, src in ((batch['obs']['low_dim']['flat_inputs'], R.r_obs), (batch['obs_next']['low_dim']['flat_inputs'], R.r_obs_next),
                     (batch['actions'], R.r_act)):
        assert torch.equal(got, src[ti])                              # gather is a pure copy
    assert torch.equal(batch['rewards'][:, 0], R.r_rew[ti]) and torch.equal(batch['dones'][:, 0], R.r_done[ti])
    L = DDPGLearner(lc, ec, sc)
    gen = torch.Generator().manual_seed(1)
    al = _layers([D, 300, 200, A], gen)
    cl = _layers([D, 400], gen) + _layers([400 + A, 300, 1], gen)
    L.model.actor.load_layers(al)
    L.model.critic.load_layers(cl)
    L.model_target.actor.load_layers(al)
    L.model_target.critic.load_layers(cl)
    O = OracleDDPGLearner(al, cl, al, cl, gamma=0.99, n_step=3, lr_actor=1e-4, lr_critic=1e-3)
    host = {k: (v['low_dim']['flat_inputs'] if isinstance(v, dict) else v) for k, v in batch.items() if k != 'indices'}
    st_o = O.optimize(host['obs'].cpu().numpy(), host['actions'].cpu().numpy(), host['rewards'].cpu().numpy().astype(np.float64),
                      host['obs_next'].cpu().numpy(), host['dones'].cpu().numpy().astype(np.float64))
    st = L.learn(batch)
    for k, v in st_o.items():
        assert abs(st[k] - v) <= 1e-5 * max(1.0, abs(v)), (k, st[k], v)
    da = torch.cat([(L.model.actor.get_layer(l)[0].cpu() - O.actor[l][0].detach()).abs().view(-1) for l in range(3)])
    dc = torch.cat([(L.model.critic.get_layer(l)[0].cpu() - O.critic[l][0].detach()).abs().view(-1) for l in range(3)])
    _assert_params_close(da, lr=1e-4, steps=1)
    _assert_params_close(dc, lr=1e-3, steps=1)


def test_fifo_conservation_at_scale():
    """configs[4]-shaped rollout (4096 actors x n 256): every completed window is either queued, sampled or
    counted as dropped; sampled windows come out in arrival order with intact payloads."""
    from surreal_b200.replay import FIFOReplay
    from surreal_b200.env import SyntheticEnv, ExpSenderWrapperMultiStepMovingWindowWithInfo as W
    N, n, D, A = 4096, 256, 16, 2
    lc, ec, sc = ppo_configs(D=D, A=A, n_step=n, stride=n, B=N, memory_size=N + 100)
    R = FIFOReplay(lc, ec, sc)
    env = SyntheticEnv(N, D, A, limit_episode_length=2 * n, seed=0)
    w = W(env, lc, sc, replay=R)
    w.reset()
    act = torch.zeros(N, A, device=DEV)
    for t in range(2 * n):
        w.stage_act[:, t % n, 0] = float(t)                       # payload marker: the step index
        w.step(act)
    st = R._read_state()
    assert st['total_in'] == 2 * N and st['count'] == N + 103 and st['dropped'] == 2 * N - (N + 103)
    b = R.sample(N)
    assert R._read_state()['count'] == 103
    first = b['actions'][:, 0, 0].cpu()
    # the oldest surviving windows are the tail of round 1 (marker 0) followed by round 2 (marker n)
    k = N - (2 * N - (N + 103))
    assert bool((first[:k] == 0).all()) and bool((first[k:] == float(n)).all())
    assert bool((b['dones'][k:, n - 1] == 1).all()) and bool((b['dones'][:, : n - 1] == 0).all())

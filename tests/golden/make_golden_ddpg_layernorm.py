#!/usr/bin/env python
"""Generate the golden vectors of the LayerNorm DDPG networks (``model.use_layernorm``) by running the REAL reference,
with the harness and generators of make_golden.py and make_golden_param_noise.py (run in the build container only):

    python tests/golden/make_golden_ddpg_layernorm.py        # writes the fixtures below

  fixture                                reference code that produced it
  -------------------------------------  ----------------------------------------------------------------------------
  ddpg_ln_optimize_{hard,soft_clipcritic}  surreal/learner/ddpg.py:186-428 with ActorNetworkX / CriticNetworkX built
  ddpg_ln_optimize_td3_double{,_reg}       with use_layernorm=True (builders.py:35-84)
  ddpg_ln_act.npz, ddpg_ln_act_ou.npz      surreal/agent/ddpg_agent.py:155-184 + action_noise.py:9-39, the same nets
  ddpg_ln_param_noise_{normal,adaptive}    surreal/agent/param_noise.py:9-74 (LayerNorm gains and biases perturbed too)

The generators are make_golden.py's own (gen_ddpg, gen_ddpg_td3, the DDPG half of gen_act, gen_act_ou) and
make_golden_param_noise.py's gen, with cfg_ddpg switched to use_layernorm=True and the fixture names prefixed.  The
harness maps torchx's LayerNorm(1) onto torch.nn.LayerNorm over the last dimension (eps 1e-5, elementwise affine,
gain 1 and bias 0 at init).  Before the first step the model's LayerNorm gains and biases are moved off (1, 0) so the
fixtures exercise them; the target nets are perturbed as in make_golden.py."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (installs the reference harness)
import make_golden_param_noise as PNG  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

H = G.H
_cfg_ddpg, _save, _construct = G.cfg_ddpg, G.save, H.construct_without_initialize


def cfg_ddpg_ln(*a, **kw):
    lc, ec, sc = _cfg_ddpg(*a, **kw)
    lc.model.use_layernorm = True
    return lc, ec, sc


def save_ln(name, **arrs):
    assert name.startswith('ddpg_'), name
    _save('ddpg_ln_' + name[len('ddpg_'):], **arrs)


def construct_ln(cls, *a, **kw):
    """The reference object, with every LayerNorm of its models moved off the (1, 0) init (seeded, own stream)."""
    obj = _construct(cls, *a, **kw)
    gen = torch.Generator().manual_seed(1234)
    for name in ('model', 'model2'):
        mdl = getattr(obj, name, None)
        if mdl is None:
            continue
        with torch.no_grad():
            for m in mdl.modules():
                if isinstance(m, torch.nn.LayerNorm):
                    m.weight.add_(0.2 * torch.randn(m.weight.shape, generator=gen))
                    m.bias.add_(0.1 * torch.randn(m.bias.shape, generator=gen))
    return obj


def gen_act():
    """The DDPG half of make_golden.gen_act (its PPO half does not depend on use_layernorm)."""
    torch.manual_seed(42)
    lc, ec, sc = G.cfg_ddpg(D=9, A=3)
    ec.num_agents = 4
    Ag = H.construct_without_initialize(G.DDPGAgent, lc, ec, sc, 3, 'training')
    obs = np.random.default_rng(43).standard_normal((5, 9)).astype(np.float32)
    np.random.seed(777)
    eps = np.stack([np.random.normal(np.zeros(3), np.ones(3)) for _ in range(5)])
    np.random.seed(777)
    acts = np.stack([Ag.act({'low_dim': {'flat_inputs': obs[i]}}) for i in range(5)])
    G.save('ddpg_act', obs=obs, unit_noise=eps, sigma=Ag.sigma, actions=acts, **G.sd_np(Ag.model, 'model/'))


def main():
    G.cfg_ddpg = PNG.G.cfg_ddpg = cfg_ddpg_ln
    G.save = PNG.save = save_ln
    H.construct_without_initialize = construct_ln
    assert G.cfg_ddpg()[0].model.use_layernorm
    G.gen_ddpg()
    G.gen_ddpg_td3()
    gen_act()
    G.gen_act_ou()
    PNG.gen('normal', 'normal')
    PNG.gen('adaptive_normal', 'adaptive')


if __name__ == '__main__':
    main()

#!/usr/bin/env python
"""Generate the golden vectors of DDPG parameter-space noise by running the REAL reference, with the harness and helpers
of make_golden.py (run in the build container only, like it):

    python tests/golden/make_golden_param_noise.py          # writes the fixtures below

  fixture                          reference code that produced it
  -------------------------------  ----------------------------------------------------------------------------------
  ddpg_param_noise_normal.npz      surreal/agent/param_noise.py:9-27 (NormalParameterNoise) through
                                   ddpg_agent.py:136-153,155-184 and ModuleDict.load (module_dict.py:47-63)
  ddpg_param_noise_adaptive.npz    param_noise.py:29-74 (AdaptiveNormalParameterNoise), the same path

Three agents (agent_id 0, 1, 2 of num_agents 3), each with its own seeded np.random stream, run 4 fetches with 23 acts
after each: param_noise.apply on the fetched numpy state dict, then ModuleDict.load, then act().  The first fetch comes
before any act (no adaptation); the adaptive distance is taken at i = 0, 10, 20, so each later mean is the distance of
act 20 divided by 23.  Every np.random.normal draw is recorded in consumption order as its N(0,1) value z (numpy's
legacy normal(loc, scale) is loc + scale * z from the same stream; the run is repeated without the recorder and must
give the same bits)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (installs the reference harness)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from surreal.distributed import ModuleDict  # noqa: E402

H = G.H
DDPGAgent, save = G.DDPGAgent, G.save
FETCHES, ACTS, AGENTS = 4, 23, 3
D, A = 9, 3


class Recorder:
    """Wraps np.random.normal: z = standard_normal(shape) from the same stream, returns loc + scale * z."""

    def __init__(self):
        self.orig = np.random.normal
        self.draws = []

    def __enter__(self):
        def normal(loc=0.0, scale=1.0, size=None):
            shape = size if size is not None else np.broadcast(np.asarray(loc), np.asarray(scale)).shape
            z = np.random.standard_normal(size=shape)
            self.draws.append(np.asarray(z, dtype=np.float64))
            return loc + scale * z
        np.random.normal = normal
        return self

    def __exit__(self, *a):
        np.random.normal = self.orig


def run_agent(kind, agent_id, versions, obs, record):
    torch.manual_seed(100 + agent_id)
    lc, ec, sc = G.cfg_ddpg(D=D, A=A)
    ec.num_agents = AGENTS
    ex = lc.algo.exploration
    ex.param_noise_type = kind
    ex.param_noise_sigma, ex.param_noise_alpha, ex.param_noise_target_stddev = 0.05, 1.15, TARGET[kind]
    Ag = H.construct_without_initialize(DDPGAgent, lc, ec, sc, agent_id, 'training')
    pn = Ag.param_noise
    np.random.seed(2000 + agent_id)
    rec = Recorder() if record else None
    out = dict(actions=[], pert=[], sigma=[], mean=[], pz=[], az=[])
    keys = None
    for f in range(FETCHES):
        params = {'ddpg': {k: v.copy() for k, v in versions[f].items()}}
        keys = list(params['ddpg'].keys())
        n0 = len(rec.draws) if rec else 0
        i_before, dist_before = getattr(pn, 'i', 0), getattr(pn, 'total_action_distance', 0.0)
        if rec:
            with rec:
                params = pn.apply(params)
        else:
            params = pn.apply(params)
        ModuleDict(Ag.module_dict()).load(params)
        out['mean'].append(float(dist_before / i_before) if i_before > 0 else np.nan)
        out['sigma'].append(float(pn.sigma))
        out['pz'].append(rec.draws[n0:] if rec else None)
        out['pert'].append({k: v.detach().numpy().copy() for k, v in Ag.model.state_dict().items() if k.startswith('actor')})
        acts, az = [], []
        for t in range(ACTS):
            n1 = len(rec.draws) if rec else 0
            if rec:
                with rec:
                    a = Ag.act({'low_dim': {'flat_inputs': obs[f, t]}})
                az.append(rec.draws[n1])
            else:
                a = Ag.act({'low_dim': {'flat_inputs': obs[f, t]}})
            acts.append(np.array(a, dtype=np.float32))
        out['actions'].append(np.stack(acts))
        out['az'].append(np.stack(az) if rec else None)
    return out, keys, float(Ag.sigma)


TARGET = {'normal': 0.005, 'adaptive_normal': 0.0055}


def gen(kind, tag):
    rng = np.random.default_rng(7 if kind == 'normal' else 8)
    torch.manual_seed(99)
    lc, ec, sc = G.cfg_ddpg(D=D, A=A)
    base = H.construct_without_initialize(DDPGAgent, lc, ec, sc, 0, 'training').model.state_dict()
    versions = []
    for f in range(FETCHES):                         # the learner's published versions: drift between fetches
        versions.append({k: (v.numpy() + 0.05 * f * rng.standard_normal(v.shape)).astype(np.float32)
                         for k, v in base.items()})
    obs = rng.standard_normal((FETCHES, ACTS, D)).astype(np.float32)
    arrs = {}
    for a in range(AGENTS):
        o, keys, act_sigma = run_agent(kind, a, versions, obs, record=True)
        o2, _, _ = run_agent(kind, a, versions, obs, record=False)
        for f in range(FETCHES):                     # the recorder did not change the stream or the arithmetic
            assert np.array_equal(o['actions'][f], o2['actions'][f])
            assert all(np.array_equal(o['pert'][f][k], o2['pert'][f][k]) for k in o['pert'][f])
        assert o['sigma'] == o2['sigma']
        arrs['a%d/actions' % a] = np.stack(o['actions'])
        arrs['a%d/action_z' % a] = np.stack(o['az'])
        arrs['a%d/sigma' % a] = np.array(o['sigma'])
        arrs['a%d/mean' % a] = np.array(o['mean'])
        arrs['a%d/action_sigma' % a] = np.float64(act_sigma)
        for f in range(FETCHES):
            assert len(o['pz'][f]) == len(keys)
            for i, z in enumerate(o['pz'][f]):
                if keys[i].startswith('actor'):      # the critic's draws are consumed but never used by the engine
                    arrs['a%d/f%d/pz/%s' % (a, f, keys[i].replace('.', '/'))] = z
            for k, v in o['pert'][f].items():
                arrs['a%d/f%d/pert/%s' % (a, f, k.replace('.', '/'))] = v
        print(tag, 'agent', a, 'sigma', o['sigma'], 'mean', o['mean'])
    for f in range(FETCHES):
        for k, v in versions[f].items():
            if k.startswith('actor'):
                arrs['f%d/model/%s' % (f, k.replace('.', '/'))] = v
    cfg = dict(kind=kind, D=D, A=A, actor_h=[20, 12], agents=AGENTS, fetches=FETCHES, acts=ACTS, sigma=0.05,
               alpha=1.15, target_stddev=TARGET[kind], interval=10, keys=keys)
    save('ddpg_param_noise_' + tag, cfg=cfg, obs=obs, **arrs)


if __name__ == '__main__':
    gen('normal', 'normal')
    gen('adaptive_normal', 'adaptive')

"""Host (numpy) and device (CUDA tensor) observations through each agent's one act entry give the same results bit for
bit, in the policy forms the host-env tests do not drive: the CNN policy of PPOAgent, QAgent with and without a state
tower, and DDPGAgent's actor forward on packed weights (the form a rollout chunk runs)."""
import numpy as np
import pytest
import torch

from helpers import ddpg_configs
from test_dqn_gpu import dqn_configs
from test_pixel_rnn_gpu import _cfg as pixel_cfg

pytestmark = pytest.mark.gpu


def _twins(make, steps, draw, act):
    """``steps`` acts of two identically seeded agents, one fed numpy and one fed device observations."""
    out = []
    for host in (True, False):
        torch.manual_seed(3)
        np.random.seed(3)
        ag = make()
        gen = torch.Generator().manual_seed(5)
        res = []
        for t in range(steps):
            x = draw(gen)
            res.append(act(ag, x.numpy() if host else x.cuda(), t))
        torch.cuda.synchronize()
        out.append((ag, res))
    return out


@pytest.mark.parametrize('mode', ['training', 'eval_deterministic', 'eval_stochastic'])
def test_ppo_cnn_policy_host_equals_device(mode):
    from surreal_b200.agent import PPOAgent
    N, A = 19, 3

    def make():
        lc, ec, sc = pixel_cfg(2, 20, 12, A, [32, 24], [28, 20], 4, N, 'clip', 1e-4, 64, 2, 6, 1, N=N)
        lc.algo.rnn.if_rnn_policy = False
        ag = PPOAgent(lc, ec, sc, 0, mode)
        ag.set_noise(np.linspace(-0.3, 0.3, N))
        return ag

    def act(ag, x, t):
        r = ag.act({'pixel': {'camera0': x}}, eps=np.full((N, A), 0.5, np.float32) if t == 2 else None)
        a, pd = (r[0], r[1][1][0]) if mode == 'training' else (r, None)
        f = lambda v: torch.as_tensor(np.asarray(v.cpu() if torch.is_tensor(v) else v, dtype=np.float32))  # noqa: E731
        return [f(a)] + ([f(pd)] if pd is not None else [])

    (h_ag, h), (d_ag, d) = _twins(make, 5, lambda g: torch.randint(0, 256, (N, 2, 20, 20), generator=g, dtype=torch.uint8),
                                  act)
    assert isinstance(h[0][0], torch.Tensor) and h[0][0].shape == (N, A)   # the CNN policy keeps the batch dimension
    for t, (x, y) in enumerate(zip(h, d)):
        for u, v in zip(x, y):
            assert torch.equal(u, v), t
    assert torch.equal(h_ag._counter, d_ag._counter)


@pytest.mark.parametrize('dueling', [True, False])
@pytest.mark.parametrize('mode', ['training', 'eval_stochastic'])
def test_dqn_host_equals_device(dueling, mode):
    from surreal_b200.agent import QAgent
    N, D, n = 33, 10, 5

    def make():
        lc, ec, sc = dqn_configs(D=D, n=n, dueling=dueling, steps=6)
        ec.num_envs = N
        return QAgent(lc, ec, sc, 0, mode)

    def act(ag, x, t):
        r = ag.act(x)
        return torch.as_tensor(r) if isinstance(r, np.ndarray) else r[1].view(-1).long().cpu()

    (h_ag, h), (d_ag, d) = _twins(make, 8, lambda g: torch.randn(N, D, generator=g), act)
    assert h[0].dtype == torch.int64
    assert len({tuple(x.tolist()) for x in h}) > 1
    for t, (x, y) in enumerate(zip(h, d)):
        assert torch.equal(x, y), t
    assert h_ag.T == d_ag.T == 8


@pytest.mark.parametrize('noise', ['normal', 'ou_noise'])
def test_ddpg_packed_forward_host_equals_device(noise):
    from surreal_b200.agent import DDPGAgent
    N, D, A = 9, 12, 4

    def make():
        lc, ec, sc = ddpg_configs(D=D, A=A, actor_h=(64, 48), critic_h=(64, 48))
        lc.algo.exploration.noise_type = noise
        ec.num_envs, ec.num_agents = N, N
        ag = DDPGAgent(lc, ec, sc, 0, 'training')
        assert ag._packed.supported
        ag._packed.refresh()
        ag._in_chunk = True                          # what a rollout chunk sets: the forward reads the packed weights
        return ag

    def act(ag, x, t):
        a = ag.act(x)
        return torch.as_tensor(a.copy()) if isinstance(a, np.ndarray) else a.cpu().clone()

    (h_ag, h), (d_ag, d) = _twins(make, 6, lambda g: torch.randn(N, D, generator=g), act)
    assert float(h[2].abs().max()) > 0.0
    for t, (x, y) in enumerate(zip(h, d)):
        assert torch.equal(x, y), t
    if noise == 'ou_noise':
        assert torch.equal(h_ag._ou_state, d_ag._ou_state)

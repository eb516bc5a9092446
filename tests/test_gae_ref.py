"""The float64 GAE reference (oracle.gae.gae_reference_fp64, a backward recurrence) against the reference formula itself
(oracle.gae.gae_from_values, a forward sum over the gamma^k / lam^k tables) run in float64, on both branches.  The GPU
envelope tests (test_gae_stats_envelope_gpu.py) measure the kernel against gae_reference_fp64, so it has to be the
same operation to float64 rounding first."""
import pytest
import torch

from oracle.gae import gae_from_values, gae_reference_fp64

GAMMA, LAM = 0.995, 0.97


def _inputs(B, n, dones, seed):
    gen = torch.Generator().manual_seed(seed)
    r = torch.randn(B, n, generator=gen, dtype=torch.float64) * 0.7 + 0.2
    v = torch.randn(B, n + 1, generator=gen, dtype=torch.float64) * 2.0
    if dones == 'random':
        d = (torch.rand(B, n, generator=gen) < 0.1).double()
    elif dones == 'first':
        d = torch.zeros(B, n, dtype=torch.float64)
        d[:, 0] = 1.0
    elif dones == 'last':
        d = torch.zeros(B, n, dtype=torch.float64)
        d[:, n - 1] = 1.0
    elif dones == 'all':
        d = torch.ones(B, n, dtype=torch.float64)
    else:
        d = torch.zeros(B, n, dtype=torch.float64)
    return r, v, d


def _check(got, exp, scale, what):
    # the two evaluation orders of the same float64 sum: ~n float64 roundings of terms bounded by ``scale``
    err = float((got - exp).abs().max())
    lim = 1e-12 * float(scale)
    assert err <= lim, '%s: %.3e > %.3e' % (what, err, lim)


@pytest.mark.parametrize('dones', ['none', 'random', 'first', 'last', 'all'])
@pytest.mark.parametrize('B,n,H', [(7, 1, None), (16, 32, None), (5, 33, None), (9, 200, None), (6, 25, 5),
                                   (4, 40, 1), (3, 50, 49), (2, 12, 12)])
def test_fp64_reference_matches_formula(B, n, H, dones):
    r, v, d = _inputs(B, n, dones, 31 * n + (H or 0))
    a64, r64 = gae_reference_fp64(r, v, d, GAMMA, LAM, horizon=H)
    a, ret = gae_from_values(r, v, d, GAMMA, LAM, horizon=H, norm_adv=False)
    E = n - (H or n) + 1
    if H is None or H == n:
        assert a64.shape == (B,) and r64.shape == (B,)
        a, ret = a.view(-1), ret.view(-1)
    else:
        assert a64.shape == (B, E) and r64.shape == (B, E)
    assert a.dtype == torch.float64 and ret.dtype == torch.float64
    scale = (r.abs().sum(1).max() + 3 * v.abs().sum(1).max())
    _check(a64, a, scale, 'adv')
    _check(r64, ret, scale, 'ret')


@pytest.mark.parametrize('scale', [0.01, 3.7])
@pytest.mark.parametrize('H', [None, 4])
def test_fp64_reference_reward_scale(scale, H):
    """reward_scale multiplies the fp32 rewards and rounds to fp32 (as the learner does) before the float64 recurrence."""
    r, v, d = _inputs(6, 20, 'random', 5)
    r32 = r.float()
    a64, r64 = gae_reference_fp64(r32, v, d, GAMMA, LAM, horizon=H, reward_scale=scale)
    rs = (r32 * scale).double()                     # fp32 product, exactly representable in float64
    a, ret = gae_from_values(rs, v, d, GAMMA, LAM, horizon=H, norm_adv=False)
    if H is None:
        a, ret = a.view(-1), ret.view(-1)
    s = rs.abs().sum(1).max() + 3 * v.abs().sum(1).max()
    _check(a64, a, s, 'adv')
    _check(r64, ret, s, 'ret')
    # and it is not the float64 product: the scaled rewards differ from r * scale in their low bits
    assert not torch.equal(rs, r32.double() * scale)


def test_fp64_reference_horizon_outputs_are_truncated_windows():
    """Output s of the horizon branch is the MLP branch of the sub-window s .. s + H - 1 (V[s + H] bootstraps)."""
    r, v, d = _inputs(5, 30, 'random', 9)
    H = 7
    a64, r64 = gae_reference_fp64(r, v, d, GAMMA, LAM, horizon=H)
    for s in range(30 - H + 1):
        # the mask of V[s] comes from done[s - 1], which lies before the sub-window: apply it to the sub-window's V[0]
        vs = v[:, s:s + H + 1].clone()
        if s > 0:
            vs[:, 0] *= 1 - d[:, s - 1]
        a, ret = gae_reference_fp64(r[:, s:s + H], vs, d[:, s:s + H], GAMMA, LAM)
        assert torch.allclose(a64[:, s], a, rtol=0, atol=1e-12) and torch.allclose(r64[:, s], ret, rtol=0, atol=1e-12)

"""Windowed GAE (sb200_gae_window_f32) on every launch path, and the PPO learner's statistics kernels in misc.cu
(reward filter, z-filter update, advantage moments + normalise, policy-distribution assembly), against float64.

GAE: every case compares adv / ret with oracle.gae.gae_reference_fp64 under a bound built from the kernel's own
roundings, printed as the ratio measured / bound:
  * td = (r + gamma V') - V: three fp32 roundings, |err| <= u (|r| + 2 gamma |V'| + |td|);
  * the two products with the fp32 gamma^k / lam^k tables, each table entry within 1 ulp (2u) of the power:
    |err| <= 6u |td gamma^k lam^k| (table entries below the fp32 normal range add at most 2^-149 each);
  * the window sum in float64 (<= H 2^-53 of the sum of |terms|) rounded once to fp32 (u |adv|);
  * the return: 3u per table product, one rounding of the sum, 2u on V[H] gamma^H (fp32 scalar), one final add.
u = 2^-24.  gamma and lam are fp32-representable here, so the learner's fp32 tables and the float64 reference take
powers of the same base.  A factor 1.001 covers the second-order (u^2) terms.  Each case also keeps the fp32-oracle bar
(BASELINE.md §5): 1e-5 max(1, rms) for raw values, 1e-5 absolute for normalised advantages.

The statistics kernels are compared with float64 evaluations of the reference formulas and, where the kernel rounds
the way torch does, bit for bit with the fp32 oracle.
"""
import math

import numpy as np
import pytest
import torch

from oracle.filters import RewardFilter as ORewardFilter
from oracle.gae import gae_from_values, gae_reference_fp64

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
U = 2.0 ** -24
U64 = 2.0 ** -53
GAMMA = float(np.float32(0.995))
LAM = float(np.float32(0.97))
# The MLP-branch kernel runs a persistent grid of at most 1056 CTAs x 8 windows (GAE_MAX_GRID in gae.cu; fewer when the
# runtime reports a lower occupancy -- the resident count itself is not measured here), so any B > 8448 makes every
# warp walk more than one window and B = 262144 at least 31: the prefetch of the next window (cur = nxt) is exercised.
MULTI_WAVE_B = (40000, 262144)


def _ops():
    from surreal_b200 import ops
    return ops


def _inputs(B, n, seed, r_mu=0.0, r_sd=0.5, v_mu=0.0, v_sd=1.0, p_done=0.05):
    gen = torch.Generator().manual_seed(seed)
    r = torch.randn(B, n, generator=gen) * r_sd + r_mu
    v = torch.randn(B, n + 1, generator=gen) * v_sd + v_mu
    d = (torch.rand(B, n, generator=gen) < p_done).float()
    if B > 2:
        d[0, 0] = 1.0              # a done at the first and at the last step of a window
        d[1, n - 1] = 1.0
    if B > 3:
        d[2] = 1.0                 # a window that is done on every step
    return r.to(DEV), v.to(DEV), d.to(DEV)


def _wsum(x, c, H):
    """sum_{j < H} c^j x[:, s + j] for every s, as a backward recurrence in float64."""
    E = x.shape[1] - H + 1
    acc = torch.zeros(x.shape[0], E, dtype=torch.float64, device=x.device)
    for k in reversed(range(H)):
        acc = x[:, k:k + E] + c * acc
    return acc


def _gae_ref_and_bound(r, v, d, H, rscale):
    """float64 adv / ret [B, E] and the per-output error bounds of the kernel (module docstring)."""
    B, n = r.shape
    a64, r64 = gae_reference_fp64(r, v, d, GAMMA, LAM, horizon=H, reward_scale=rscale)
    if a64.dim() == 1:
        a64, r64 = a64.view(-1, 1), r64.view(-1, 1)
    rs = (r * rscale).double() if rscale != 1.0 else r.double()
    vm = v.double().clone()
    vm[:, 1:] *= 1 - d.double()
    td = rs + GAMMA * vm[:, 1:] - vm[:, :-1]
    e_td = U * (rs.abs() + 2 * GAMMA * vm[:, 1:].abs() + td.abs())
    abs_t = _wsum(td.abs(), GAMMA * LAM, H)
    tiny = H * 2.0 ** -149 * (1.0 + float(td.abs().max()))
    b_adv = 1.001 * (_wsum(e_td + 6 * U * td.abs(), GAMMA * LAM, H) + H * U64 * abs_t + U * a64.abs() + tiny)
    abs_r = _wsum(rs.abs(), GAMMA, H)
    r_sum = _wsum(rs, GAMMA, H)
    E = n - H + 1
    boot = (GAMMA ** H) * vm[:, H:H + E].abs()
    b_ret = 1.001 * ((3 * U + H * U64) * abs_r + U * r_sum.abs() + 2 * U * boot + U * r64.abs())
    return a64, r64, b_adv, b_ret


def _norm_ref_and_bound(a64, b_adv, one_pass):
    """float64 (adv - mean) / std (unbiased) and the bound of the kernel's normalised advantages, given the bound b_adv
    of its raw ones.  mean and std are computed in float64 from the fp32 advantages and rounded to fp32 (u each); the
    std of perturbed values moves by at most the rms of the perturbation; (a - mean) and the division round once each.
    one_pass: the large-batch path's variance (Q - S^2 / B) / (B - 1), whose float64 cancellation adds
    <= 4 B 2^-53 Q / (B - 1) to the variance."""
    N = a64.numel()
    mu, sig = a64.mean(), a64.std()
    assert float(sig) > 1e-3, 'the batch must be above the 1e-4 std floor'
    z = (a64 - mu) / sig
    e_rms = float(b_adv.pow(2).mean().sqrt()) * math.sqrt(N / (N - 1))
    d_mu = float(b_adv.mean()) + U * abs(float(mu)) + N * U64 * float(a64.abs().mean())
    var_err = (4 * N * U64 * float(a64.pow(2).sum()) / (N - 1)) if one_pass else 2 * N * U64 * float(sig) ** 2
    d_sig = e_rms + var_err / (2 * float(sig)) + U * float(sig)
    bound = 1.001 * ((b_adv + d_mu + U * (a64 - mu).abs()) / sig + z.abs() * (d_sig / float(sig) + U))
    return z, bound


def _ratio(got, ref, bound):
    return float(((got.double() - ref).abs() / bound).max())


def _oracle32(r, v, d, H, rscale, norm):
    rs = r * rscale if rscale != 1.0 else r
    a, ret = gae_from_values(rs.cpu(), v.cpu(), d.cpu(), GAMMA, LAM, horizon=H, norm_adv=norm)
    return a.view(r.shape[0], -1), ret.view(r.shape[0], -1)


def _bar_raw(got, exp, what):
    got, exp = got.detach().cpu().double(), exp.detach().cpu().double()
    err, lim = float((got - exp).abs().max()), 1e-5 * max(1.0, float(exp.pow(2).mean().sqrt()))
    assert err <= lim, '%s vs fp32 oracle: %.3e > %.3e' % (what, err, lim)


def _bar_norm(got, exp, what):
    err = float((got.detach().cpu().double() - exp.detach().cpu().double()).abs().max())
    assert err <= 1e-5, '%s vs fp32 oracle: %.3e > 1e-5' % (what, err)


def _check_gae(tag, r, v, d, H=None, norm=False, rscale=1.0, ws=None, oracle=True):
    """Run the kernel and hold it to the float64 bound and the fp32-oracle bar; returns (adv, ret)."""
    ops = _ops()
    B, n = r.shape
    Hn = n if H is None else H
    adv, ret = ops.gae_window(r, v, d, GAMMA, LAM, horizon=H, norm_adv=norm, reward_scale=rscale, ws=ws)
    torch.cuda.synchronize()
    assert adv.shape == (B, n - Hn + 1) and ret.shape == adv.shape
    a64, r64, b_adv, b_ret = _gae_ref_and_bound(r, v, d, Hn, rscale)
    q_ret = _ratio(ret, r64, b_ret)
    if norm:
        z, b_z = _norm_ref_and_bound(a64, b_adv, one_pass=(Hn == n and B > 16384))
        q_adv = _ratio(adv, z, b_z)
    else:
        q_adv = _ratio(adv, a64, b_adv)
    print('measured gae %s: adv %.3f ret %.3f of the bound' % (tag, q_adv, q_ret))
    assert q_adv <= 1.0 and q_ret <= 1.0, (tag, q_adv, q_ret)
    if oracle:
        e_adv, e_ret = _oracle32(r, v, d, Hn, rscale, norm)
        (_bar_norm if norm else _bar_raw)(adv, e_adv, tag + ' adv')
        _bar_raw(ret, e_ret, tag + ' ret')
    return adv, ret


# -- the MLP branch: register windows (n = 32, 64, 128, 256) and the generic loop ----------------------------------------

@pytest.mark.parametrize('n,B,norm', [
    (32, 1, False), (32, 1000, False), (32, MULTI_WAVE_B[0], False), (32, MULTI_WAVE_B[1], False),
    (32, MULTI_WAVE_B[1], True),
    (64, 5000, False), (64, 5000, True),
    (128, 1, False), (128, 3000, True), (128, MULTI_WAVE_B[0], False), (128, MULTI_WAVE_B[1], False),
    (256, 3000, False), (256, 3000, True),
    (1, 5000, False), (1, 5000, True), (33, 2000, True), (200, 1500, False), (200, 20000, False),
    (6144, 64, False), (6144, 64, True),
])
def test_gae_full_path(n, B, norm):
    r, v, d = _inputs(B, n, 7 * n + B)
    _check_gae('n=%d B=%d norm=%d' % (n, B, norm), r, v, d, norm=norm)


@pytest.mark.parametrize('n', [32, 128])
def test_gae_window_independent_of_batch(n):
    """Un-normalised, window b of a B = 262144 call (a later window of its warp, loaded while the previous one was
    reduced) is bit-identical to the same window computed in a call of 64 windows (each the first of its warp)."""
    ops = _ops()
    B = MULTI_WAVE_B[1]
    r, v, d = _inputs(B, n, 100 + n)
    adv, ret = ops.gae_window(r, v, d, GAMMA, LAM, norm_adv=False)
    adv_s, ret_s = torch.empty_like(adv), torch.empty_like(ret)
    for b0 in range(0, B, 64):
        ops.gae_window(r[b0:b0 + 64], v[b0:b0 + 64], d[b0:b0 + 64], GAMMA, LAM, norm_adv=False,
                       adv=adv_s[b0:b0 + 64], ret=ret_s[b0:b0 + 64])
    torch.cuda.synchronize()
    bad = int((adv != adv_s).sum()) + int((ret != ret_s).sum())
    print('measured gae batch independence n=%d: %d differing outputs of %d' % (n, bad, 2 * B))
    assert bad == 0


# -- advantage normalisation on both sides of the large-batch switch ----------------------------------------------------

@pytest.mark.parametrize('B', [16384, 16385])
@pytest.mark.parametrize('offset', [0.0, 100.0])
def test_gae_norm_mode_switch(B, offset):
    """B <= 16384: the last CTA normalises alone (two-pass float64).  B > 16384: per-CTA float64 partials, a one-pass
    variance in the last CTA and gae_normalize_kernel.  offset 100: rewards of order 100 with a spread of 0.5 and small
    values, so the advantages share a common offset of ~2500 and the one-pass variance cancels most of its digits."""
    n = 64
    r, v, d = _inputs(B, n, B + int(offset), r_mu=offset, v_sd=1.0 if offset == 0 else 0.1,
                      p_done=0.05 if offset == 0 else 0.0)
    tag = 'norm B=%d offset=%g' % (B, offset)
    if offset == 0:
        _check_gae(tag, r, v, d, norm=True)
        return
    # With a common offset mu, rounding mu to fp32 moves every normalised advantage by up to ulp(mu) / std ~ 1e-4, in the
    # fp32 oracle as in the kernel: the 1e-5 bar cannot hold between them (torch's fp32 mean and the float64 mean rounded
    # to fp32 differ in about a third of such batches).  This case is held to the float64 bound, which carries that term.
    raw, _ = _ops().gae_window(r, v, d, GAMMA, LAM, norm_adv=False)
    a = raw.double().view(-1)
    assert float(a.mean()) > 300 * float(a.std())
    _check_gae(tag, r, v, d, norm=True, oracle=False)


def test_gae_workspace_reuse_across_modes():
    """One workspace through large-batch, fused, horizon, then large-batch normalisation again: the self-resetting
    ticket counter leaves every call correct and the repeated call bit-identical."""
    from surreal_b200 import _lib
    ws = torch.zeros(int(_lib.lib().sb200_gae_workspace_bytes(1, 1, 1)), dtype=torch.uint8, device=DEV)
    big = _inputs(20000, 64, 1)
    a1, r1 = _check_gae('ws mode 2', *big, norm=True, ws=ws)
    _check_gae('ws mode 1', *_inputs(3000, 33, 2), norm=True, ws=ws)
    _check_gae('ws horizon', *_inputs(500, 40, 3), H=8, norm=True, ws=ws)
    a2, r2 = _check_gae('ws mode 2 again', *big, norm=True, ws=ws, oracle=False)
    assert torch.equal(a1, a2) and torch.equal(r1, r2)


@pytest.mark.parametrize('rscale', [1.0, 0.01, 3.7])
@pytest.mark.parametrize('path', ['register', 'generic', 'horizon'])
def test_gae_reward_scale(path, rscale):
    """reward_scale multiplies the fp32 rewards (rounded to fp32) before everything else, on each path."""
    n, B, H = {'register': (128, 3000, None), 'generic': (200, 1000, None), 'horizon': (60, 700, 9)}[path]
    r, v, d = _inputs(B, n, 11 + n, r_sd=1.0, r_mu=0.3)
    _check_gae('%s scale=%g' % (path, rscale), r, v, d, H=H, rscale=rscale)


# -- the horizon (RNN) kernel ---------------------------------------------------------------------------------------------

def _horizon_n_max(H_of_n):
    """The largest n whose per-CTA shared memory (2H + 8 (3n + 1)) * 4 B fits the kernel's 200 KB."""
    n = 1
    while (2 * H_of_n(n + 1) + 8 * (3 * (n + 1) + 1)) * 4 <= 200 * 1024:
        n += 1
    return n


HZ_H1, HZ_H5, HZ_HN1 = (lambda n: 1), (lambda n: 5), (lambda n: n - 1)


@pytest.mark.parametrize('n,H,B,norm', [
    (50, 1, 200, False), (50, 5, 200, True), (50, 49, 200, False), (50, 49, 200, True),
    (_horizon_n_max(HZ_H1), 1, 16, False), (_horizon_n_max(HZ_H5), 5, 9, True), (_horizon_n_max(HZ_HN1), None, 33, True),
    (200, 5, 5120, True),                 # normalisation over B E = 1 003 520 outputs by one CTA
])
def test_gae_horizon(n, H, B, norm):
    H = n - 1 if H is None else H
    r, v, d = _inputs(B, n, 3 * n + H)
    _check_gae('horizon n=%d H=%d B=%d norm=%d' % (n, H, B, norm), r, v, d, H=H, norm=norm)


# -- limits: the largest accepted window runs and is right, one past it is refused before any launch ---------------------

@pytest.mark.parametrize('path,n,H', [
    ('full', 6144, None),                                  # 2n fp32 tables <= 48 KB
    ('horizon H=1', _horizon_n_max(HZ_H1), 1),
    ('horizon H=n-1', _horizon_n_max(HZ_HN1), _horizon_n_max(HZ_HN1) - 1),
])
def test_gae_limits(path, n, H):
    from surreal_b200 import _lib
    ops = _ops()
    _check_gae('limit %s n=%d' % (path, n), *_inputs(8, n, n), H=H)
    n1 = n + 1
    H1 = None if H is None else (1 if H == 1 else n1 - 1)
    r, v, d = _inputs(8, n1, n1)
    E = n1 - (H1 or n1) + 1
    adv = torch.full((8, E), 7.0, device=DEV)
    ret = torch.full((8, E), 7.0, device=DEV)
    torch.cuda.synchronize()
    before = _lib.call_counter_kernels()
    with pytest.raises(_lib.SB200Error, match='invalid argument'):
        ops.gae_window(r, v, d, GAMMA, LAM, horizon=H1, norm_adv=True, adv=adv, ret=ret)
    torch.cuda.synchronize()
    assert _lib.call_counter_kernels() == before, 'refused call launched a kernel'
    assert bool((adv == 7.0).all()) and bool((ret == 7.0).all())


def test_gae_single_window_normalised():
    """B = 1 with norm_adv: the reference divides by std() of one element (NaN) and returns NaN.  The kernel's NaN std
    falls to the 1e-4 floor and the one advantage normalises to exactly 0 (DESIGN.md, numerics); the return is unchanged."""
    for n in (32, 200):
        r, v, d = _inputs(1, n, n)
        adv, ret = _ops().gae_window(r, v, d, GAMMA, LAM, norm_adv=True)
        torch.cuda.synchronize()
        e_adv, e_ret = _oracle32(r, v, d, n, 1.0, True)
        assert bool(torch.isnan(e_adv).all())
        assert float(adv) == 0.0
        _bar_raw(ret, e_ret, 'B=1 ret')


# -- reward filter (misc.cu reward_filter_kernel) --------------------------------------------------------------------------

RF_EPS = 1e-5


def _reward_filter(x, stats, scale):
    from surreal_b200 import _lib, ops
    out = torch.empty_like(x)
    _lib.check(_lib.lib().sb200_reward_filter_f32(ops._ptr(x), x.numel(), float(scale), RF_EPS, ops._ptr(stats),
                                                  ops._ptr(out), ops._stream()), 'sb200_reward_filter_f32')
    torch.cuda.synchronize()
    return out


def _rf_fp32(xs, cnt, s, q):
    """The reference's forward in fp32 with the kernel's floor: fmax keeps eps where sqrt of a negative variance is NaN."""
    mean = s / cnt
    std = torch.fmax((q / cnt - mean.pow(2)).pow(0.5), torch.tensor(RF_EPS, dtype=torch.float32))
    return torch.clamp((xs - mean) / std, -5.0, 5.0)


def _rf_rewards(n, call, mu, seed):
    if n == 1:                             # one reward per call: an alternating sequence keeps the variance positive
        return torch.tensor([mu + (2.0 if call % 2 == 0 else -2.0)])
    gen = torch.Generator().manual_seed(seed + call)
    r = torch.randn(n, generator=gen) + mu
    if call == 0:
        r[0] = 0.0                         # the first call's only output that is not clamped to +-5
    return r


@pytest.mark.parametrize('n', [1, 1023, 1024, 1025, 131072])
@pytest.mark.parametrize('mu,scale', [(0.0, 1.0), (0.0, 0.37), (0.25, 1.0), (0.1, 2.5)])
def test_reward_filter_sequence(n, mu, scale):
    """12 calls: out = clamp((x - mean) / max(std, eps), +-5) with the statistics before the call, x = r * scale
    rounded to fp32; then count += n, sum += sum(x), sumsq = sum(x^2) (overwritten: the reference's quirk).
    Each call: outputs against the float64 evaluation of that formula (bound below) and bit for bit against the fp32
    oracle; the statistics against float64 sums rounded once to fp32 (<= 1 ulp: the two float64 summation orders)."""
    stats = torch.tensor([RF_EPS, 0.0, 0.0], dtype=torch.float32, device=DEV)
    worst = 0.0
    for call in range(12):
        r = _rf_rewards(n, call, mu, 1000 * n)
        x = r * np.float32(scale)                        # what the kernel filters: fp32 product
        before = stats.cpu()
        out = _reward_filter(r.to(DEV), stats, scale).cpu()
        cnt, s, q = before[0], before[1], before[2]
        if call == 0:                                    # count = eps, variance 0: every output is +-5 or 0
            assert bool(((out.abs() == 5.0) | (x.abs() < 5 * RF_EPS)).all())
            assert n == 1 or float(out[0]) == 0.0
        # bit for bit with the fp32 oracle (the variance is an fp32 product then an fp32 subtraction, like torch's)
        orf = ORewardFilter(RF_EPS)
        orf.count, orf.running_sum, orf.running_sumsq = cnt.clone(), s.clone(), q.clone()
        exp32 = orf.forward(x)
        assert torch.equal(out, exp32), ('call %d differs from the fp32 oracle' % call)
        # float64 formula on the same statistics
        c64, s64, q64 = float(cnt), float(s), float(q)
        m64 = s64 / c64
        var = q64 / c64 - m64 * m64
        if call > 0:
            e_var = U * (q64 / c64) * 2 + 3 * U * m64 * m64 + U * abs(var)     # q / c, m (then m^2), the difference
            assert var > 8 * e_var, ('the test data must stay in the finite regime', call, var, e_var)
            sd = max(math.sqrt(var), RF_EPS)
            e_sd = sd * (e_var / (2 * var) + U) if math.sqrt(var) > RF_EPS else 0.0
            xd = x.double()
            z = (xd - m64) / sd
            ref = z.clamp(-5.0, 5.0)
            bound = 1.001 * ((U * abs(m64) + U * (xd - m64).abs()) / sd + z.abs() * (e_sd / sd + U)) + 1e-300
            worst = max(worst, float(((out.double() - ref).abs() / bound).max()))
        # statistics: count in fp32, sum += fp32(float64 sum), sumsq = fp32(float64 sum of fp32 squares)
        after = stats.cpu()
        t_s = np.float32(x.double().sum())
        t_q = np.float32((x * x).double().sum())
        assert float(after[0]) == float(np.float32(np.float32(cnt) + np.float32(n)))
        exp_s = np.float32(np.float32(s) + t_s)
        assert abs(float(after[1]) - float(exp_s)) <= float(np.spacing(max(abs(exp_s), abs(t_s)))), (call, after, exp_s)
        assert abs(float(after[2]) - float(t_q)) <= float(np.spacing(abs(t_q))), (call, after, t_q)
    print('measured reward filter n=%d mu=%g scale=%g: %.3f of the bound' % (n, mu, scale, worst))
    assert worst <= 1.0


@pytest.mark.parametrize('n', [1, 1025])
def test_reward_filter_negative_variance(n):
    """Rewards with mean 1 and spread 0.1: with sumsq overwritten by the last batch, sumsq / count - mean^2 < 0 from the
    third call on.  The reference's sqrt(negative) is NaN and its clamp(NaN, min=eps) keeps it, so it returns NaN rewards.
    The kernel floors the std at eps instead (fmaxf drops the NaN) and returns clamp((x - mean) / eps, +-5): finite
    rewards, an intended deviation (DESIGN.md, numerics).  Pinned bit for bit."""
    stats = torch.tensor([RF_EPS, 0.0, 0.0], dtype=torch.float32, device=DEV)
    negative = 0
    for call in range(6):
        gen = torch.Generator().manual_seed(call)
        r = torch.randn(n, generator=gen) * 0.1 + 1.0
        before = stats.cpu()
        out = _reward_filter(r.to(DEV), stats, 1.0).cpu()
        cnt, s, q = before[0], before[1], before[2]
        orf = ORewardFilter(RF_EPS)
        orf.count, orf.running_sum, orf.running_sumsq = cnt.clone(), s.clone(), q.clone()
        ref = orf.forward(r)
        assert bool(torch.isfinite(out).all())
        assert torch.equal(out, _rf_fp32(r, cnt, s, q))
        if call >= 2:
            assert float(q / cnt - (s / cnt).pow(2)) < 0
            assert bool(torch.isnan(ref).all())
            assert torch.equal(out, torch.clamp((r - s / cnt) / RF_EPS, -5.0, 5.0))
            negative += 1
        else:
            assert torch.equal(out, ref)
    assert negative == 4


# -- z-filter statistics (misc.cu zfilter_update_kernel) -------------------------------------------------------------------

@pytest.mark.parametrize('D,rows,layout', [
    (1, 1000000, 'dense'), (3, 1000000, 'window'), (3, 4097, 'dense'), (64, 1000000, 'dense'),
    (64, 100000, 'window'), (1000, 20000, 'dense'), (1000, 3000, 'window'),
])
def test_zfilter_update(D, rows, layout):
    """stats = sum[D] | sumsq[D] | count, four calls.  The kernel's contract is a float64 sum per call (of x, and of the
    fp32 squares x*x) rounded once to fp32 and added in fp32 -- not torch's fp32 reduction order.  Strides as the learner
    passes them: 'dense' is _xraw_eff (rows padded to a multiple of 4 columns), 'window' the first observation of each
    [n + 1, D] window record (ldx = (n + 1) D)."""
    ops = _ops()
    n = 8
    stats = torch.cat([torch.zeros(D), torch.full((D,), 1e-5), torch.tensor([1e-5])]).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(D + rows)
    worst = 0.0
    for call in range(4):
        if layout == 'dense':
            ld = (D + 3) // 4 * 4
            full = torch.randn(rows, ld, generator=gen, device=DEV) * 2.0 + 3.0
            x, ldx = full[:, :D], ld
        else:
            full = torch.randn(rows, n + 1, D, generator=gen, device=DEV) * 2.0 + 3.0
            x, ldx = full[:, 0], (n + 1) * D
        prev = stats.double().cpu()
        ops.zfilter_update(full, rows, D, ldx, stats)
        torch.cuda.synchronize()
        got = stats.cpu()
        t_s = x.double().sum(0).float().cpu()
        t_q = (x * x).double().sum(0).float().cpu()
        exp_s = (prev[:D].float() + t_s)
        exp_q = (prev[D:2 * D].float() + t_q)
        tol_s = torch.tensor(np.spacing(np.maximum(exp_s.abs().numpy(), t_s.abs().numpy())))
        tol_q = torch.tensor(np.spacing(np.maximum(exp_q.abs().numpy(), t_q.abs().numpy())))
        es = float(((got[:D] - exp_s).abs() / tol_s).max())
        eq = float(((got[D:2 * D] - exp_q).abs() / tol_q).max())
        worst = max(worst, es, eq)
        assert float(got[2 * D]) == float(np.float32(np.float32(prev[2 * D]) + np.float32(rows)))
    print('measured zfilter D=%d rows=%d %s: %.3f ulp at most' % (D, rows, layout, worst))
    assert worst <= 1.0


# -- advantage moments + normalise (the data-parallel learner's global-batch normalisation) ---------------------------------

@pytest.mark.parametrize('N', [1, 2, 1024, 1025, 262144])
def test_moments_normalize_match_fused(N):
    """sb200_moments_f32 + sb200_normalize_f32 on one rank against GAE's own fused normalisation (fused two-pass for
    N <= 16384, the large-batch path above): within 1e-5 absolute, and both against float64.  N = 1: both give 0."""
    from surreal_b200 import _lib
    ops = _ops()
    L = _lib.lib()
    r, v, d = _inputs(N, 32, N)
    raw, _ = ops.gae_window(r, v, d, GAMMA, LAM, norm_adv=False)
    fused, _ = ops.gae_window(r, v, d, GAMMA, LAM, norm_adv=True)
    x = raw.clone().view(-1)
    mom = torch.zeros(3, dtype=torch.float64, device=DEV)
    _lib.check(L.sb200_moments_f32(ops._ptr(x), N, ops._ptr(mom), ops._stream()), 'sb200_moments_f32')
    _lib.check(L.sb200_normalize_f32(ops._ptr(x), N, ops._ptr(mom), 1e-4, ops._stream()), 'sb200_normalize_f32')
    torch.cuda.synchronize()
    assert float(mom[2]) == N
    if N == 1:
        assert float(x) == 0.0 and float(fused) == 0.0
        return
    err = float((x - fused.view(-1)).abs().max())
    a = raw.double().view(-1)
    z64 = (a - a.mean()) / a.std()
    e64 = float((x.double() - z64).abs().max())
    print('measured moments+normalize N=%d: %.3e vs fused, %.3e vs float64' % (N, err, e64))
    assert err <= 1e-5 and e64 <= 1e-5


# -- policy-distribution assembly (misc.cu make_pd_kernel) -----------------------------------------------------------------

@pytest.mark.parametrize('B,A,noise', [(1, 1, False), (37, 6, True), (1024, 8, True), (300, 17, False)])
def test_make_pd(B, A, noise):
    """pd[b] = [mean[b] | exp(log_var) * exp(log_noise[b])] into padded rows (ldp > 2A) from a padded mean (ldm > A):
    bit for bit with torch.exp on the device composed the same way (both are the CUDA library's expf), within 2 ulp of
    the float64 exp (expf's documented bound; 4.5 ulp for the rounded product of two), and the padding untouched."""
    ops = _ops()
    gen = torch.Generator(device=DEV).manual_seed(B * A)
    mean_full = torch.randn(B, A + 5, generator=gen, device=DEV)
    mean = mean_full[:, 2:2 + A]
    log_var = torch.randn(A, generator=gen, device=DEV) * 2.0
    log_noise = (torch.rand(B, generator=gen, device=DEV) - 0.5) if noise else None
    pd_full = torch.full((B, 2 * A + 3), 9.0, device=DEV)
    pd = pd_full[:, :2 * A]
    ops.make_pd(mean, log_var, B, A, pd, log_noise=log_noise)
    torch.cuda.synchronize()
    std = torch.exp(log_var).expand(B, A)
    if noise:
        std = std * torch.exp(log_noise).view(B, 1)
    assert torch.equal(pd[:, :A], mean)
    assert torch.equal(pd[:, A:], std)
    assert bool((pd_full[:, 2 * A:] == 9.0).all())
    e64 = torch.exp(log_var.double()).expand(B, A)
    if noise:
        e64 = e64 * torch.exp(log_noise.double()).view(B, 1)
    ulp = torch.tensor(np.spacing(e64.float().abs().cpu().numpy()), device=DEV).double()
    q = float(((pd[:, A:].double() - e64).abs() / ulp).max())
    print('measured make_pd B=%d A=%d noise=%d: %.2f ulp of the float64 exp' % (B, A, noise, q))
    assert q <= (4.5 if noise else 2.0)

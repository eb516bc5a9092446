"""The one-launch PPO learner kernel (csrc/epoch2.cu) epoch by epoch: every state it carries from one epoch to the next
inside a launch, checked against float64 and against itself.

A rig binds two FlatNets, their MlpTrainers and EpochKernel blocks the way PPOLearner._epoch_kernels does (z-filter on,
x read with the window stride (n + 1) D, stop flag, statistics and gradient-norm slices, lr and hyper-parameters as
device tensors) and drives EpochPair directly.  Before every launch the scratch the kernel owns is filled with NaN, so
a value it fails to write shows.  S_k is the state after k one-epoch launches from S_0:

1. each one-epoch launch k against float64 at S_{k-1}: gradients, gradient norms, the z-filtered input, the Adam step
   (bit for bit against sb200_clip_adam_f32) and the loss statistics; lr / clip_eps / beta change between launches;
2. one launch of k epochs ends in S_k bit for bit (W2^T refresh, x_in cache, step count, last-epoch gradient);
3. the results are the same bit for bit at every grid, in particular in adapt mode, whose backward reloads the
   activations from global memory when a CTA holds more than one row block;
4. the KL early stop lands on the right epoch and leaves exactly that epoch's policy; a stop flag raised before the
   launch leaves the policy alone and still trains the value network;
5. the above at both sides of every width, head, row and row-split edge, and at the plan's limits (found by bisection).

Bars quote the worst value measured on an H100 80GB HBM3 next to them."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

import grad_ref as R
from surreal_b200 import _lib, ops
from test_epoch_plan import _plan_sms, largest_rows, widest_square
from test_grads_gpu import E2_BAR, GN_BAR, _check_grads, _clear_relu_ties, _layers
from test_mlp_forward_envelope_gpu import _zfilter64

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NAN = float('nan')
EPS = 1e-5                    # z-filter std floor
N_WIN = 3                     # window steps per record: x rows are (N_WIN + 1) D apart, actions N_WIN A, behaviour 2 N_WIN A
ETA = 250.0
TIE = 2e-5                    # float64 pre-activations this close to 0 take the kernel's relu
ST = dict(SURR=0, LOSS=1, ENTROPY=2, KL_PRE=3, KL_POST=4, GN_ACTOR=5, VAL_LOSS=6, EXPL_VAR=7, GN_CRITIC=8, RET_MEAN=9,
          EPOCHS=14, VAL_MOMENTS=16)
# Relative error of each statistic against float64 (relative to max(|value|, 1e-3)), bar after the measured worst:
# SURR 8.0e-6, LOSS 2.0e-5 (adapt, the hinge term), ENTROPY 3.5e-7, KL_PRE 1.9e-6, KL_POST 2.6e-6, VAL_LOSS 8.0e-8,
# EXPL_VAR 7.0e-6, RET_MEAN 4.5e-8; the VAL_MOMENTS (hi + lo) pairs: mean(ret - v) 1.1e-6, mean((ret - v)^2) 8.7e-8,
# mean(ret) 1.2e-15, mean(ret^2) 1.3e-15 (float64 sums of float32 returns).  Other bars: gradients per tensor, worst
# relative L2 / max error 6.5e-6 / 8.3e-6 (E2_BAR = 3e-5); gradient norms 6.8e-6 (GN_BAR = 1e-5); x_in 0.46 of the
# float32 filter's rounding bound.  The Adam step, one launch against chained launches and the grids: bit for bit.
STAT_BAR = dict(SURR=4e-5, LOSS=1e-4, ENTROPY=2e-6, KL_PRE=1e-5, KL_POST=1e-5, VAL_LOSS=4e-7, EXPL_VAR=3e-5,
                RET_MEAN=2e-7, MOM_D=5e-6, MOM_D2=4e-7, MOM_R=1e-14, MOM_R2=1e-14)
WORST = {}


def _record(name, v):
    WORST[name] = max(WORST.get(name, 0.0), v)


def _f64layers(net, buf):
    return [tuple(t.double() for t in net.get_layer(l, buf=buf)) for l in range(net.n_layers)]


def _masks(layers, x64, h_kernel):
    """Per hidden layer: float64's own relu, except the units whose float64 pre-activation is within TIE of 0, which
    take the kernel's saved fp32 activation (h_kernel; None: no such unit may exist).  -> masks, units borrowed."""
    masks, borrowed, h = [], 0, x64
    for l, (w, b) in enumerate(layers[:-1]):
        pre = F.linear(h, w, b)
        m = pre > 0
        near = pre.abs() < TIE
        if h_kernel is None:
            assert not bool(near.any()), 'a relu tie at a state without saved activations'
        else:
            m = torch.where(near, h_kernel[l][:, :pre.shape[1]] > 0, m)
            borrowed += int(near.sum())
        masks.append(m.double())
        h = pre * masks[-1]
    return masks, borrowed


def _pin(col):
    """Column ``col`` of raw inputs -> 0.75 + 4e-6 j, |j| <= 12 (idempotent): with the statistics below its variance is
    exactly 0, so the filter divides by the std floor eps and the values land within +-4.8, unclamped."""
    def f(t):
        t = t.clone()
        c = t[:, col]
        near = (c - 0.75).abs() < 1e-4
        j = torch.where(near, torch.round((c - 0.75) / 4e-6), torch.round(c * 5.0)).clamp(-12, 12)
        t[:, col] = (0.75 + 4e-6 * j).float()
        return t
    return f


class State:
    def __init__(self, tr):
        self.p, self.m, self.v, self.ws = (t.clone() for t in (tr.net.params, tr.exp_avg, tr.exp_avg_sq, tr.ws))

    def load(self, tr):
        for src, dst in zip((self.p, self.m, self.v, self.ws), (tr.net.params, tr.exp_avg, tr.exp_avg_sq, tr.ws)):
            dst.copy_(src)

    def equal(self, o):
        return all(torch.equal(a, b) for a, b in zip((self.p, self.m, self.v, self.ws), (o.p, o.m, o.v, o.ws)))


class Rig:
    """Actor ``ad`` (mode 0 clip / 1 adapt) and critic ``cd`` on M rows.  ``aclip`` / ``cclip`` = (clip mode, clip value
    as a multiple of the float64 S_0 gradient norm (mode 1) or largest entry (mode 2), weight decay).  ``ref_shift``: the
    reference policy's mean sits that many stds from the current one (0: KL(ref || policy) starts at 0).  ``hinge``:
    adapt mode's kl_target puts the pre-step KL at 2x (True) or 0.5x (False) the hinge's branch point."""

    def __init__(self, ad, cd, M, mode, seed, lr=1e-3, splits=None, aclip=(1, 10.0, 0.0), cclip=(0, 0.0, 0.0),
                 ref_shift=0.2, hinge=True, grid=None):
        gen = torch.Generator().manual_seed(seed)
        D, A = ad[0], ad[-1]
        assert cd[0] == D and cd[-1] == 1
        self.D, self.A, self.M, self.mode = D, A, M, mode
        al, cl = _layers(ad, gen), _layers(cd, gen)
        # narrower policies for wide heads: at std 0.5 a 32-dimensional likelihood is below the 1e-5 clamp on most rows
        log_var = torch.full((1, A), -0.7 if A <= 8 else -1.6) + 0.2 * torch.rand(1, A, generator=gen)
        cnt, zc = 256, min(3, D - 1)
        smp = torch.randn(cnt, D, generator=gen, dtype=torch.float64) * 1.3 + 0.2
        zs = torch.cat([smp.sum(0), (smp * smp).sum(0), torch.tensor([float(cnt)], dtype=torch.float64)])
        zs[zc], zs[D + zc] = 0.75 * cnt, 0.5625 * cnt                    # variance exactly 0
        zs = zs.float()
        pin = _pin(zc)
        tf = lambda t: R.zfilter(pin(t), zs)  # noqa: E731
        # ties cleared at twice TIE: the kernel's own filtered input differs from float64's by rounding
        x = pin(_clear_relu_ties(torch.randn(M, D, generator=gen) * 1.3 + 0.2, [(al, tf), (cl, tf)], tol=2 * TIE, gen=gen))
        self.x_raw = x.to(DEV)
        self.zs = zs.to(DEV)
        with torch.no_grad():
            mean = torch.tanh(R.trunk(tf(x), [(R.f64(w), R.f64(b)) for w, b in al]))
        std = torch.exp(R.f64(log_var)).expand(M, A)
        g64 = lambda *sh: torch.randn(*sh, generator=gen, dtype=torch.float64)  # noqa: E731
        bm = (mean + 0.3 * std * g64(M, A)).clamp(-0.99, 0.99)
        bs = std * torch.exp(0.2 * g64(M, 1))
        self.actions = (bm + 0.5 * bs * g64(M, A)).float().to(DEV)
        self.behave = torch.cat([bm, bs], 1).float().to(DEV)
        self.ref = torch.cat([mean + ref_shift * std * g64(M, A), std], 1).float().to(DEV)
        self.adv, self.ret = torch.randn(M, generator=gen).to(DEV), torch.randn(M, generator=gen).to(DEV)
        kl0 = float(R.kl(R.f64(self.ref[:, :A]).cpu(), R.f64(self.ref[:, A:]).cpu(), mean, std).mean())
        self.kl_target = max(kl0, 1e-6) / 2 * (0.5 if hinge else 2.0)
        # window-layout device buffers: step 0 holds the batch, the other steps NaN
        xw = torch.full((M, N_WIN + 1, D), NAN, device=DEV)
        xw[:, 0] = self.x_raw
        aw = torch.full((M, N_WIN, A), NAN, device=DEV)
        aw[:, 0] = self.actions
        bw = torch.full((M, N_WIN, 2 * A), NAN, device=DEV)
        bw[:, 0] = self.behave
        self._bufs = (xw, aw, bw)
        self.an = ops.FlatNet(ad, [ops.ACT_RELU, ops.ACT_RELU, ops.ACT_TANH], DEV, extra=A).load_layers(al, extra=log_var)
        self.cn = ops.FlatNet(cd, [ops.ACT_RELU, ops.ACT_RELU, ops.ACT_NONE], DEV).load_layers(cl)
        self.at = ops.MlpTrainer(self.an, M, lr, clip_mode=aclip[0], clip_value=1.0, weight_decay=aclip[2], splits=splits)
        self.ct = ops.MlpTrainer(self.cn, M, lr, clip_mode=cclip[0], clip_value=1.0, weight_decay=cclip[2], splits=splits)
        self.stats = torch.zeros(32, device=DEV)
        self.stop = torch.zeros(1, dtype=torch.int32, device=DEV)
        self.hyper = torch.tensor([0.2, 1.0], dtype=torch.float64, device=DEV)
        self.lr0 = lr
        self.pk = ops.EpochKernel(self.at, mode, xw, (N_WIN + 1) * D, M, self.zs, EPS, self.stats, 1,
                                  norm_out=self.stats[ST['GN_ACTOR']:ST['GN_ACTOR'] + 1], stop_flag=self.stop, actions=aw,
                                  lda=N_WIN * A, adv=self.adv, behave_pd=bw, ldb=N_WIN * 2 * A, ref_pd=self.ref, ldr=2 * A,
                                  hyper=self.hyper, eta=ETA, kl_target=self.kl_target, stop_threshold=0.0, grid=grid)
        self.vk = ops.EpochKernel(self.ct, 2, xw, (N_WIN + 1) * D, M, self.zs, EPS, self.stats, 1,
                                  norm_out=self.stats[ST['GN_CRITIC']:ST['GN_CRITIC'] + 1], returns=self.ret)
        assert ops.EpochPair.supported(self.pk, self.vk), (ad, cd, M)
        self.pair = ops.EpochPair(self.pk, self.vk)
        self.solo = None
        # clip values relative to the float64 gradient at S_0
        x64 = R.zfilter(self.x_raw, self.zs)
        r = self.ref_policy(self.an.params, x64, None)
        rv = R.value(_f64layers(self.cn, self.cn.params), x64, self.ret)
        for k, (mode_, f, _), gs in ((self.pk, aclip, r['grads'] + [(r['g_log_var'],)]), (self.vk, cclip, rv['grads'])):
            flat = torch.cat([g.reshape(-1) for wb in gs for g in wb])
            k.args.clip_value = float(f * (flat.norm() if mode_ == 1 else flat.abs().max())) if mode_ else 0.0
        self.s0 = self.state()

    # -- state -------------------------------------------------------------------------------------------------
    def state(self):
        return State(self.at), State(self.ct)

    def load(self, st):
        st[0].load(self.at)
        st[1].load(self.ct)
        self.stats.zero_()
        self.stop.zero_()

    def set_hyper(self, k):
        """lr, clip_eps and beta of launch k (k = 0: the defaults), written in place as the learner does."""
        self.at.lr.fill_(self.lr0 * (1.0 + 0.25 * k))
        self.ct.lr.fill_(self.lr0 * (1.0 - 0.05 * k))
        self.hyper.copy_(torch.tensor([0.2 - 0.01 * k, 1.0 + 0.5 * k], dtype=torch.float64))

    # -- launches ----------------------------------------------------------------------------------------------
    def _poison(self, pair):
        s = ops.EpochPair.plan(pair.policy, pair.value)['s']
        jobs = [(self.at, True, s[0])] + ([(self.ct, False, s[1])] if pair.value is not None else [])
        for tr, policy, sj in jobs:
            net = tr.net
            for t in [tr.x_in, tr.grad] + tr.h + tr.d:
                t.fill_(NAN)
            for z in range(sj):
                for l in range(net.n_layers):
                    net.W(l, tr.slabs[z]).fill_(NAN)
                    net.b(l, tr.slabs[z])[:net.layout[l]['N']].fill_(NAN)
            if policy:
                net.extra_view(tr.slabs[0]).fill_(NAN)
        pair.ws.fill_(255)

    def run(self, p_epochs, v_epochs=None, threshold=0.0, solo=False):
        """One launch: the policy for p_epochs, the value network for v_epochs (None: the same) or not at all (solo)."""
        if solo and self.solo is None:
            self.solo = ops.EpochPair(self.pk, None)
        pair = self.solo if solo else self.pair
        self.pk.args.epochs = p_epochs
        self.vk.args.epochs = p_epochs if v_epochs is None else v_epochs
        self.pk.args.stop_threshold = threshold
        self._poison(pair)
        pair.run()
        torch.cuda.synchronize()

    def ref_policy(self, params, x64, masks):
        hv = self.hyper.tolist()
        layers = _f64layers(self.an, params)
        lv = self.an.extra_view(params).double()
        if self.mode == 0:
            return R.ppo_policy(layers, lv, x64, self.actions, self.adv, self.behave, 'clip', masks=masks, clip_eps=hv[0])
        return R.ppo_policy(layers, lv, x64, self.actions, self.adv, self.behave, 'adapt', masks=masks, ref=self.ref,
                            beta=hv[1], kl_target=self.kl_target, eta=ETA)

    def kl64(self, params, x64):
        A = self.A
        with torch.no_grad():
            mean = torch.tanh(R.trunk(x64, _f64layers(self.an, params)))
        std = torch.exp(self.an.extra_view(params).double()).expand_as(mean)
        return float(R.kl(R.f64(self.ref[:, :A]), R.f64(self.ref[:, A:]), mean, std).mean())


def _padding_zero(tr, what):
    """FlatNet's contract: the padding columns of W, the padding of every bias and of the extra block stay exactly 0."""
    net = tr.net
    for name, buf in (('params', net.params), ('exp_avg', tr.exp_avg), ('exp_avg_sq', tr.exp_avg_sq), ('grad', tr.grad)):
        for l, lay in enumerate(net.layout):
            N = lay['N']
            assert not bool(net.W(l, buf)[:, N:].any()) and not bool(net.b(l, buf)[N:].any()), (what, name, l)
        if net.extra:
            assert not bool(buf[net.extra_off + net.extra:].any()), (what, name, 'extra')


def _stat(got, exp, name, what):
    err = abs(float(got) - float(exp)) / max(abs(float(exp)), 1e-3)
    _record('stat ' + name, err)
    assert err <= STAT_BAR[name], (what, name, float(got), float(exp), err)


def _check_launch(rig, k, s_prev, s_next, h_prev, what):
    """One-epoch launch k took s_prev (S_{k-1}) to s_next (S_k); the trainers hold what it left."""
    at, ct, M, D = rig.at, rig.ct, rig.M, rig.D
    # the z-filtered input, against float64 within the float32 filter's rounding bound
    sx = at.x_in[:, :D].double()
    z, ez = _zfilter64(rig.x_raw.double(), rig.zs)
    assert bool(((sx - z).abs() <= ez).all()), (what, k, 'x_in', float(((sx - z).abs() / ez).max()))
    assert torch.equal(ct.x_in, at.x_in) and not bool(at.x_in[:, D:].any()), (what, k, 'x_in padding')
    _record('x_in / bound', float(((sx - z).abs() / ez).max()))
    # gradients at S_{k-1} on the kernel's own input; relu ties take the kernel's activations of that state
    pl, cl = _f64layers(rig.an, s_prev[0].p), _f64layers(rig.cn, s_prev[1].p)
    pm, pb = _masks(pl, sx, h_prev)
    cm, cb = _masks(cl, sx, ct.h)
    assert pb + cb <= 1e-3 * M * (sum(rig.an.dims[1:3]) + sum(rig.cn.dims[1:3])), (what, k, pb, cb)
    r = rig.ref_policy(s_prev[0].p, sx, pm)
    rv = R.value(cl, sx, rig.ret, masks=cm)
    _check_grads(rig.an, at.grad, r['grads'], '%s actor k=%d' % (what, k), extra=r['g_log_var'], bar=E2_BAR)
    _check_grads(rig.cn, ct.grad, rv['grads'], '%s critic k=%d' % (what, k), bar=E2_BAR)
    st = rig.stats.double()
    na = math.sqrt(sum(float(g.pow(2).sum()) for wb in r['grads'] for g in wb) + float(r['g_log_var'].pow(2).sum()))
    nc = math.sqrt(sum(float(g.pow(2).sum()) for wb in rv['grads'] for g in wb))
    for got, exp, nm in ((st[ST['GN_ACTOR']], na, 'actor'), (st[ST['GN_CRITIC']], nc, 'critic')):
        assert exp > 0.0, (what, k, nm, 'a zero gradient tests nothing')
        _record('gradnorm', abs(float(got) - exp) / exp)
        assert abs(float(got) - exp) <= GN_BAR * exp, (what, k, nm, float(got), exp)
    # Adam: sb200_clip_adam_f32 from S_{k-1} with the kernel's gradient and workspace gives S_k bit for bit
    for tr, blk, sp, sn in ((at, rig.pk, s_prev[0], s_next[0]), (ct, rig.vk, s_prev[1], s_next[1])):
        p, m, v, ws = sp.p.clone(), sp.m.clone(), sp.v.clone(), tr.ws.clone()
        a = blk.args
        _lib.check(_lib.lib().sb200_clip_adam_f32(C.c_void_p(p.data_ptr()), C.c_void_p(tr.grad.data_ptr()), C.c_void_p(m.data_ptr()),
                                                  C.c_void_p(v.data_ptr()), p.numel(), C.c_void_p(tr.lr.data_ptr()), 0.9, 0.999,
                                                  1e-8, a.weight_decay, a.clip_mode, a.clip_value, C.c_void_p(ws.data_ptr()),
                                                  None, None, ops._stream()), 'sb200_clip_adam_f32')
        torch.cuda.synchronize()
        assert torch.equal(p, sn.p) and torch.equal(m, sn.m) and torch.equal(v, sn.v), (what, k, 'adam', a.mode)
        assert torch.equal(ws, sn.ws) and torch.equal(ws, tr.ws), (what, k, 'workspace')
    # statistics
    _stat(st[ST['SURR']], r['surr'], 'SURR', what)
    _stat(st[ST['LOSS']], r['loss'], 'LOSS', what)
    _stat(st[ST['ENTROPY']], r['entropy'], 'ENTROPY', what)
    if rig.mode == 1:
        _stat(st[ST['KL_PRE']], r['kl'], 'KL_PRE', what)
        assert abs(float(r['kl']) - 2 * rig.kl_target) > 1e-2 * 2 * rig.kl_target, (what, k, 'hinge branch point')
    kl_post = rig.kl64(s_next[0].p, sx)
    _stat(st[ST['KL_POST']], kl_post, 'KL_POST', what)
    assert float(st[ST['EPOCHS']]) == 1.0, (what, k, float(st[ST['EPOCHS']]))
    _stat(st[ST['VAL_LOSS']], rv['loss'], 'VAL_LOSS', what)
    _stat(st[ST['EXPL_VAR']], rv['explained_var'], 'EXPL_VAR', what)
    _stat(st[ST['RET_MEAN']], rv['ret_mean'], 'RET_MEAN', what)
    d, rr = R.f64(rig.ret).reshape(-1, 1) - rv['v'], R.f64(rig.ret)
    mom = st[ST['VAL_MOMENTS']:ST['VAL_MOMENTS'] + 8].view(4, 2).sum(1)
    for i, (nm, exp) in enumerate((('MOM_D', d.mean()), ('MOM_D2', d.pow(2).mean()), ('MOM_R', rr.mean()), ('MOM_R2', rr.pow(2).mean()))):
        _stat(mom[i], exp, nm, what)
    return float(rig.stats[ST['KL_POST']])


def epochwise(rig, E, vary=False, check=True, what=''):
    """E one-epoch launches from S_0 (each checked against float64 when ``check``); -> states [S_0 .. S_E], the
    gradients and statistics each launch left, and the post-step KL of each epoch as the kernel reported it."""
    rig.load(rig.s0)
    rig.set_hyper(0)
    states, grads, stats, kls = [rig.s0], [None], [None], [None]
    h_prev = None
    for k in range(1, E + 1):
        if vary:
            rig.set_hyper(k)
        rig.stats.zero_()
        rig.run(1)
        states.append(rig.state())
        grads.append((rig.at.grad.clone(), rig.ct.grad.clone()))
        stats.append(rig.stats.clone())
        kls.append(_check_launch(rig, k, states[k - 1], states[k], h_prev, what) if check else float(rig.stats[ST['KL_POST']]))
        h_prev = [h.clone() for h in rig.at.h[:2]]                  # the trailing forward: activations at S_k
    for tr in (rig.at, rig.ct):
        _padding_zero(tr, what)
    rig.set_hyper(0)
    return states, grads, stats, kls


def _same(rig, st_pair, grads, what):
    got = rig.state()
    assert got[0].equal(st_pair[0]), (what, 'policy state')
    assert got[1].equal(st_pair[1]), (what, 'value state')
    if grads is not None:
        assert torch.equal(rig.at.grad, grads[0]) and torch.equal(rig.ct.grad, grads[1]), (what, 'grad')


def one_launch_equals_chained(rig, states, grads, stats, pairs, what):
    """Launches of (policy epochs, value epochs) from S_0 end where the chained one-epoch launches did."""
    E = len(states) - 1
    for p, v in pairs:
        rig.load(rig.s0)
        rig.run(p, v)
        got = rig.state()
        assert got[0].equal(states[p][0]), (what, p, v, 'policy state after one launch != chained launches')
        assert got[1].equal(states[v][1]), (what, p, v, 'value state after one launch != chained launches')
        assert torch.equal(rig.at.grad, grads[p][0]) and torch.equal(rig.ct.grad, grads[v][1]), (what, p, v, 'grad')
        assert float(rig.stats[ST['EPOCHS']]) == p, (what, p, float(rig.stats[ST['EPOCHS']]))
        sp, sv = stats[p], stats[v]
        for name in ('SURR', 'LOSS', 'ENTROPY', 'KL_PRE', 'KL_POST', 'GN_ACTOR'):
            assert torch.equal(rig.stats[ST[name]], sp[ST[name]]), (what, p, v, name)
        for i in list(range(ST['VAL_LOSS'], ST['RET_MEAN'] + 1)) + list(range(ST['VAL_MOMENTS'], ST['VAL_MOMENTS'] + 8)):
            assert torch.equal(rig.stats[i], sv[i]), (what, p, v, i)
        assert p <= E and v <= E
    _padding_zero(rig.at, what)
    _padding_zero(rig.ct, what)


def _report():
    print('measured worst:', ', '.join('%s %.2e' % kv for kv in sorted(WORST.items())))


# ---- 1 + 2 + 4 at the bench shape ------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def bench():
    """configs[1]'s networks on a 1024-row batch, clip mode, the reference policy equal to the starting one (KL from 0),
    the actor's gradient clipped by norm, the critic unclipped: ten chained one-epoch launches checked against float64."""
    rig = Rig([64, 256, 256, 8], [64, 256, 256, 1], 1024, 0, seed=1, lr=3e-3, aclip=(1, 0.5, 0.0), cclip=(0, 0.0, 0.0),
              ref_shift=0.0)
    out = epochwise(rig, 10, check=True, what='bench')
    _report()
    return rig, out


def test_bench_shape_epoch_by_epoch_against_float64(bench):
    rig, (states, grads, stats, kls) = bench
    assert len(states) == 11
    one_launch_equals_chained(rig, states, grads, stats, [(10, 10), (3, 5), (5, 3), (1, 10)], 'bench')


def test_policy_only_launch_equals_chained(bench):
    """EpochPair(policy, None): its plan differs from the pair's (more row splits), so the chain is its own."""
    rig = bench[0]
    rig.load(rig.s0)
    chain = []
    for k in range(4):
        rig.run(1, solo=True)
        chain.append((State(rig.at), rig.at.grad.clone()))
    rig.load(rig.s0)
    v0 = State(rig.ct)
    rig.run(4, solo=True)
    assert State(rig.at).equal(chain[-1][0]) and torch.equal(rig.at.grad, chain[-1][1])
    assert State(rig.ct).equal(v0), 'a policy-only launch touched the value network'
    assert float(rig.stats[ST['EPOCHS']]) == 4.0


def _threshold(kls, e):
    """A stop threshold that the post-step KL of epoch e exceeds and no earlier one reaches, 1 % clear of both."""
    below = max(kls[1:e], default=0.0)
    if not (kls[e] > 1.0201 * below and kls[e] > 0.0):
        return None
    return math.sqrt(kls[e] * below) if below > 0 else kls[e] / 1.02


def test_kl_early_stop_at_the_threshold(bench):
    rig, (states, grads, stats, kls) = bench
    E = 6
    later = [e for e in range(2, E) if _threshold(kls, e) is not None]
    assert later, kls
    for e in (1, later[-1]):
        thr = _threshold(kls, e)
        assert thr is not None, (e, kls)
        rig.load(rig.s0)
        rig.run(E, threshold=thr)
        assert float(rig.stats[ST['EPOCHS']]) == e, (e, float(rig.stats[ST['EPOCHS']]), kls)
        assert int(rig.stop.item()) == 1
        assert float(rig.stats[ST['KL_POST']]) == kls[e], (e, float(rig.stats[ST['KL_POST']]), kls[e])
        assert State(rig.at).equal(states[e][0]) and torch.equal(rig.at.grad, grads[e][0]), ('policy after the stop', e)
        assert State(rig.ct).equal(states[E][1]) and torch.equal(rig.ct.grad, grads[E][1]), ('value after the stop', e)
    # a stop flag raised before the launch: the policy is left alone, the value network trains
    rig.load(rig.s0)
    rig.stop.fill_(1)
    rig.run(E)
    assert State(rig.at).equal(rig.s0[0]) and float(rig.stats[ST['EPOCHS']]) == 0.0
    assert State(rig.ct).equal(states[E][1]) and torch.equal(rig.ct.grad, grads[E][1])
    assert int(rig.stop.item()) == 1


# ---- 1 with the device hyper-parameters changing between launches, clip modes 0 / 1 / 2, weight decay -------------
HYPER_CASES = [
    # (actor dims, critic dims, rows, mode, aclip, cclip, hinge)
    ([17, 300, 200, 6], [17, 100, 68, 1], 1000, 1, (2, 0.3, 1e-3), (1, 10.0, 1e-4), True),
    ([17, 300, 200, 6], [17, 100, 68, 1], 200, 1, (1, 0.5, 0.0), (2, 0.3, 0.0), False),
    ([24, 64, 48, 32], [24, 64, 48, 1], 515, 0, (0, 0.0, 1e-2), (1, 0.5, 1e-3), True),
]


@pytest.mark.parametrize('case', range(len(HYPER_CASES)))
def test_epoch_by_epoch_with_changing_hyper_parameters(case):
    ad, cd, M, mode, aclip, cclip, hinge = HYPER_CASES[case]
    rig = Rig(ad, cd, M, mode, seed=20 + case, lr=2e-3, aclip=aclip, cclip=cclip, hinge=hinge)
    epochwise(rig, 4, vary=True, what='hyper%d' % case)
    _report()


# ---- 3: grid invariance --------------------------------------------------------------------------------------------
def _grids(G):
    return [G] + [g for g in (68, 37, 7, 1) if g < G]


@pytest.mark.parametrize('mode', [0, 1])
def test_results_do_not_depend_on_the_grid(mode):
    """Three policy and four value epochs at every grid.  Adapt mode: with 2 n_rb <= G row blocks (one per CTA) the
    backward uses the activations the forward left in shared memory, with more it reloads them; both must agree."""
    G = _plan_sms()
    M = 16 * (G // 2) - 5 if mode == 1 else 1024                     # adapt: n_items = 2 n_rb <= G at the full grid
    rig = Rig([64, 256, 256, 8], [64, 256, 256, 1], M, mode, seed=40 + mode)
    n_items = 2 * ((M + 15) // 16)
    ref = None
    for g in _grids(G):
        rig.pk.args.grid = g
        assert ops.EpochPair.plan(rig.pk, rig.vk)['grid'] == g
        rig.load(rig.s0)
        rig.run(3, 4)
        got = (rig.state(), rig.at.grad.clone(), rig.ct.grad.clone(), rig.stats.clone())
        if ref is None:
            ref = got
            if mode == 1:
                assert n_items <= g, (n_items, g)
            continue
        assert got[0][0].equal(ref[0][0]) and got[0][1].equal(ref[0][1]), ('state', g)
        assert torch.equal(got[1], ref[1]) and torch.equal(got[2], ref[2]), ('grad', g)
        assert torch.equal(got[3], ref[3]), ('stats', g, (got[3] != ref[3]).nonzero().view(-1).tolist())
    assert mode == 0 or n_items > 68


# ---- 5: the shape envelope -----------------------------------------------------------------------------------------
# (id, actor dims, critic dims, rows, mode, trainer splits): widths = 1 / 3 mod 4 and 15 / 16 / 17 (16-row blocks), 256
# against 257 / 260 (the 64-quad passes of the GEMMs), heads 1 4 5 8 9 31 32 (the head's second column quad), rows 2 3 15
# 16 17 64 65 and thousands, row splits 1 2 3 and 9 with ragged last splits and empty / short dW3 block ranges.
ENVELOPE = [
    ('w17-15-17-h5', [17, 15, 17, 5], [17, 16, 15, 1], 65, 0, None),
    ('w3-257-260-h9', [3, 257, 260, 9], [3, 256, 257, 1], 17, 1, None),
    ('w16-256-257-h31', [16, 256, 257, 31], [16, 260, 256, 1], 64, 0, None),
    ('w15-260-256-h32', [15, 260, 256, 32], [15, 17, 16, 1], 16, 1, None),
    ('w13-16-15-h1-m2', [13, 16, 15, 1], [13, 15, 17, 1], 2, 0, None),
    ('w5-17-16-h4-m3', [5, 17, 16, 4], [5, 16, 16, 1], 3, 1, None),
    ('w1-33-31-h8-m15', [1, 33, 31, 8], [1, 31, 33, 1], 15, 0, None),
    ('s2-ragged', [17, 64, 48, 6], [17, 48, 64, 1], 2017, 1, 2),
    ('s3-ragged', [17, 64, 48, 6], [17, 48, 64, 1], 3001, 0, 3),
    ('s9-empty-dw3', [16, 16, 16, 4], [16, 16, 16, 1], 577, 1, 9),
    ('s9-ragged', [16, 16, 16, 4], [16, 16, 16, 1], 1000, 0, 9),
    ('m4096', [64, 256, 256, 8], [64, 256, 256, 1], 4096, 1, None),
]


def _run_envelope(ad, cd, M, mode, splits, what, E=3):
    rig = Rig(ad, cd, M, mode, seed=sum(ad) + M, lr=2e-3, splits=splits, aclip=(1, 10.0, 0.0), cclip=(1, 10.0, 0.0))
    pl = ops.EpochPair.plan(rig.pk, rig.vk)
    states, grads, stats, _ = epochwise(rig, E, what=what)
    one_launch_equals_chained(rig, states, grads, stats, [(E, E), (E - 1, E), (E, 1)], what)
    _report()
    return pl


@pytest.mark.parametrize('case', ENVELOPE, ids=[c[0] for c in ENVELOPE])
def test_envelope(case):
    what, ad, cd, M, mode, splits = case
    pl = _run_envelope(ad, cd, M, mode, splits, what)
    if splits is not None:                                           # the row split the case is named for
        assert pl['s'][0] == splits and pl['s'][1] == splits, pl
        assert M % pl['rps'][0] != 0, pl                              # a ragged last split
        n_rb, s = (M + 15) // 16, splits
        per = -(-n_rb // s)                                          # dW3 sums row blocks [z per, (z + 1) per)
        if 'empty' in what:
            assert per * (s - 1) >= n_rb, (per, n_rb)
        elif s < 9:
            assert n_rb < per * s, (per, n_rb)                       # a short last range


def test_plan_limits_run_and_the_next_shape_falls_back():
    """At the largest batch the plan takes for the bench shape, the widest square hidden layers at 1024 rows and that
    width's largest batch: two epochs against float64 and as one launch.  One row or one unit more is rejected, and
    PPOLearner then takes the launch chain."""
    from helpers import ppo_configs
    from surreal_b200.learner import PPOLearner
    m_bench, h = largest_rows(), widest_square()
    m_wide = largest_rows(h, h)
    for what, dims, M in (('bench M max', 256, m_bench), ('H max', h, 1024), ('H max, M max', h, m_wide)):
        _run_envelope([64, dims, dims, 8], [64, dims, dims, 1], M, 0 if dims == 256 else 1, None, what, E=2)
    for B, h_, taken in ((m_bench, 256, True), (m_bench + 1, 256, False), (1024, h + 1, False)):
        lc, ec, sc = ppo_configs(D=64, A=8, actor_h=(h_, h_), critic_h=(h_, h_), n_step=2, stride=2, B=B)
        L = PPOLearner(lc, ec, sc)
        assert (L._epoch_kernels() is not None) == taken and (L._ek[3] is not None) == taken, (B, h_)
        del L

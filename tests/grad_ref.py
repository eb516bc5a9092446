"""Float64 autograd references of the training losses: the loss, its statistics and the gradient with respect to
every parameter, the head pre-activation and log_var.  The arithmetic is the oracle's (oracle/pd.py, oracle/ppo.py
_clip_loss / _adapt_loss / _value_update, oracle/ddpg.py, oracle/nets.py), restated over float64 copies so that the
kernels' fp32 gradients can be held to a tight bar.

Layers are ``[(W [out, in], b [out])]`` (torch.nn.Linear convention); every function detaches and copies its inputs,
so callers may pass fp32 tensors from any device.  Policies are rows ``[mean(A) | std(A)]``."""
import math

import torch
import torch.nn.functional as F

_LOG_2PI = math.log(2.0 * math.pi)
_LOG_2PIE = math.log(2.0 * math.pi * math.e)


def f64(t):
    return torch.as_tensor(t).detach().to(torch.float64).clone()


def _leaves(layers):
    return [(f64(w).requires_grad_(True), f64(b).requires_grad_(True)) for w, b in layers]


def _flat(layers):
    return [t for wb in layers for t in wb]


def _pairs(gs):
    return [(gs[i], gs[i + 1]) for i in range(0, len(gs), 2)]


def zfilter(x, stats, eps=1e-5):
    """oracle/filters.py ZFilter.forward; ``stats`` = [running_sum(D) | running_sumsq(D) | count]."""
    x, stats = f64(x), f64(stats)
    D = x.shape[-1]
    cnt = stats[2 * D]
    mean = stats[:D] / cnt
    std = torch.clamp((stats[D:2 * D] / cnt - mean.pow(2)).pow(0.5), min=eps)
    return torch.clamp((x - mean) / std, -5.0, 5.0)


def trunk(x, layers, aux=None, aux_layer=-1, masks=None):
    """Linear-ReLU-...-Linear (no final activation); ``aux`` is concatenated to the input of layer ``aux_layer``
    (the DDPG critic's action columns, oracle/nets.py ddpg_critic).  ``masks[i]`` (0/1, one per hidden layer) replaces
    relu's own test: a kernel's saved activations then decide units whose pre-activation rounds to either side of 0."""
    h = x
    for i, (w, b) in enumerate(layers):
        if i == aux_layer:
            h = torch.cat((h, aux), 1)
        h = F.linear(h, w, b)
        if i < len(layers) - 1:
            h = torch.relu(h) if masks is None else h * f64(masks[i]).to(h.device)
    return h


def hidden_margin(x, layers, aux=None, aux_layer=-1):
    """Per row, the smallest |pre-activation| over the hidden units: rows where it is tiny can flip a relu between fp32
    and fp64."""
    h, m = f64(x), None
    for i, (w, b) in enumerate(layers[:-1]):
        if i == aux_layer:
            h = torch.cat((h, f64(aux)), 1)
        h = F.linear(h, f64(w).to(h.device), f64(b).to(h.device))
        r = h.abs().min(dim=1)[0]
        m = r if m is None else torch.minimum(m, r)
        h = torch.relu(h)
    return m


def loglikelihood(a, mean, std):
    quad = (((a - mean) / std) ** 2).sum(dim=1, keepdim=True)
    return -0.5 * quad - 0.5 * _LOG_2PI * a.shape[1] - std.log().sum(dim=1, keepdim=True)


def likelihood(a, mean, std):
    return torch.clamp(loglikelihood(a, mean, std).exp(), min=1e-5)


def kl(m0, s0, m1, s1):
    """KL(p0 || p1) per row."""
    return (s1 / s0).log().sum(dim=1) + ((s0 ** 2 + (m0 - m1) ** 2) / (2.0 * s1 ** 2)).sum(dim=1) - 0.5 * m0.shape[1]


def _policy_loss(pre, log_var, actions, adv, behave, mode, clip_eps=0.2, ref=None, beta=1.0, kl_target=0.015, eta=250.0):
    """_clip_loss (mode 'clip') / _adapt_loss (mode 'adapt') of oracle/ppo.py on the head pre-activation ``pre``."""
    A = pre.shape[1]
    mean = torch.tanh(pre)
    std = torch.exp(log_var).reshape(1, A).expand_as(mean)
    bm, bs = behave[:, :A], behave[:, A:]
    adv = adv.reshape(-1, 1)
    st = {'entropy': (0.5 * std.log().sum(dim=1) + 0.5 * _LOG_2PIE * A).mean()}
    if mode == 'clip':
        ratio = likelihood(actions, mean, std) / likelihood(actions, bm, bs)
        surr = -ratio * adv
        csurr = -torch.clamp(ratio, 1 - clip_eps, 1 + clip_eps) * adv
        loss = torch.cat([surr, csurr], 1).max(1)[0].mean()
        st['surr'] = surr.mean()
        st['ratio'] = ratio.view(-1)
    else:
        prob_behave = likelihood(actions, bm, bs)
        klm = kl(ref[:, :A], ref[:, A:], mean, std).mean()
        surr = -(adv * (likelihood(actions, mean, std) / torch.clamp(prob_behave, min=1e-2))).mean()
        loss = surr + beta * klm
        st['hinge'] = bool(klm.item() - 2.0 * kl_target > 0)
        if st['hinge']:
            loss = loss + eta * (klm - 2.0 * kl_target).pow(2)
        st['surr'] = surr
        st['kl'] = klm
    st['loss'] = loss
    return loss, st


def _result(loss, st, leaves, named):
    gs = torch.autograd.grad(loss, leaves, allow_unused=True)
    out = {k: (v.detach() if torch.is_tensor(v) else v) for k, v in st.items()}
    for k, g in zip(named, gs):
        out[k] = g
    return out


def policy_loss_head(pre, log_var, actions, adv, behave, mode, **hyper):
    """Loss kernels alone: gradients w.r.t. the head pre-activation (``g_pre``) and log_var (``g_log_var``)."""
    pre, lv = f64(pre).requires_grad_(True), f64(log_var).reshape(-1).requires_grad_(True)
    ref = hyper.pop('ref', None)
    loss, st = _policy_loss(pre, lv, f64(actions), f64(adv), f64(behave), mode,
                            ref=f64(ref) if ref is not None else None, **hyper)
    return _result(loss, st, [pre, lv], ['g_pre', 'g_log_var'])


def ppo_policy(layers, log_var, x, actions, adv, behave, mode, masks=None, **hyper):
    """One policy update's loss on the actor ``layers`` over (already whitened) inputs ``x``: ``grads`` per layer,
    ``g_log_var``, ``g_pre``, plus the loss statistics.  ``masks`` as in trunk."""
    L = _leaves(layers)
    lv = f64(log_var).reshape(-1).requires_grad_(True)
    pre = trunk(f64(x), L, masks=masks)
    ref = hyper.pop('ref', None)
    loss, st = _policy_loss(pre, lv, f64(actions), f64(adv), f64(behave), mode,
                            ref=f64(ref) if ref is not None else None, **hyper)
    out = _result(loss, st, _flat(L) + [lv, pre], ['_g%d' % i for i in range(2 * len(L))] + ['g_log_var', 'g_pre'])
    out['grads'] = _pairs([out.pop('_g%d' % i) for i in range(2 * len(L))])
    return out


def value(layers, x, ret, masks=None):
    """_value_update's loss mean((v - ret)^2) and explained variance; ``grads`` per layer, ``g_pre`` = dL/dv, ``v``.
    ``masks`` as in trunk."""
    L = _leaves(layers)
    v = trunk(f64(x), L, masks=masks)
    ret = f64(ret).reshape(-1, 1)
    loss = (v - ret).pow(2).mean()
    st = {'loss': loss, 'explained_var': 1 - torch.var(ret - v) / torch.var(ret), 'ret_mean': ret.mean(), 'v': v}
    out = _result(loss, st, _flat(L) + [v], ['_g%d' % i for i in range(2 * len(L))] + ['g_pre'])
    out['grads'] = _pairs([out.pop('_g%d' % i) for i in range(2 * len(L))])
    return out


def lstm(x, h0, c0, w_ih, w_hh, b_ih, b_hh):
    """One torch.nn.LSTM layer (batch_first, gate order i, f, g, o) as a plain cell loop, differentiable: no copies, so
    callers pass float64 leaves.  x [B, L, D]; h0 / c0 [B, H] or None (zeros).  -> dict: ``h`` / ``c`` [B, L, H] (the
    output and cell sequences), ``gates`` [B, L, 4H] (activated: sigmoid i, f, o and tanh g), ``pre`` (list of L
    [B, 4H] gate pre-activations, to take gradients with respect to), ``h_last`` / ``c_last`` [B, H]."""
    B, L, _ = x.shape
    H = w_hh.shape[1]
    h = x.new_zeros(B, H) if h0 is None else h0
    c = x.new_zeros(B, H) if c0 is None else c0
    hs, cs, gs, pres = [], [], [], []
    for t in range(L):
        pre = F.linear(x[:, t], w_ih, b_ih) + F.linear(h, w_hh, b_hh)
        i, f, g, o = torch.sigmoid(pre[:, :H]), torch.sigmoid(pre[:, H:2 * H]), torch.tanh(pre[:, 2 * H:3 * H]), \
            torch.sigmoid(pre[:, 3 * H:])
        c = f * c + i * g
        h = o * torch.tanh(c)
        pres.append(pre)
        gs.append(torch.cat((i, f, g, o), 1))
        hs.append(h)
        cs.append(c)
    return {'h': torch.stack(hs, 1), 'c': torch.stack(cs, 1), 'gates': torch.stack(gs, 1), 'pre': pres, 'h_last': h,
            'c_last': c}


def _rnn_features(stem, x, h0, c0, zs):
    """z-filter (``zs`` = its statistics, or None: off) -> LSTM from the DETACHED initial cells (ppo.py:507-510) -> rows
    b*L + t.  ``stem`` = (w_ih, w_hh, b_ih, b_hh) float64 leaves."""
    x = f64(x)
    if zs is not None:
        x = zfilter(x, zs)
    B, L = x.shape[:2]
    r = lstm(x, None if h0 is None else f64(h0).to(x.device), None if c0 is None else f64(c0).to(x.device), *stem)
    return r['h'].reshape(B * L, -1)


def rnn_features(stem, x, h0, c0, zs=None):
    """The head input of RNN mode in float64, without gradients: rows b*L + t of the LSTM outputs."""
    with torch.no_grad():
        return _rnn_features([f64(t) for t in stem], x, h0, c0, zs)


_STEM_NAMES = ['g_w_ih', 'g_w_hh', 'g_b_ih', 'g_b_hh']


def ppo_policy_rnn(stem, layers, log_var, x, h0, c0, actions, adv, behave, mode, zs=None, masks=None, **hyper):
    """RNN mode's policy loss (ppo.py:507-556): raw observations x [B, L, D] -> z-filter -> LSTM from (h0, c0) -> actor
    head -> loss, over the B*L rows b*L + t.  ``grads`` per head layer, ``g_log_var``, ``stem`` = the gradients of
    (W_ih, W_hh, b_ih, b_hh) in torch's layout, ``g_pre`` and the loss statistics.  ``masks`` as in trunk."""
    S = [f64(t).requires_grad_(True) for t in stem]
    L = _leaves(layers)
    lv = f64(log_var).reshape(-1).requires_grad_(True)
    pre = trunk(_rnn_features(S, x, h0, c0, zs), L, masks=masks)
    A = pre.shape[1]
    ref = hyper.pop('ref', None)
    loss, st = _policy_loss(pre, lv, f64(actions).reshape(-1, A), f64(adv).reshape(-1), f64(behave).reshape(-1, 2 * A),
                            mode, ref=f64(ref).reshape(-1, 2 * A) if ref is not None else None, **hyper)
    nl = 2 * len(L)
    out = _result(loss, st, _flat(L) + [lv, pre] + S, ['_g%d' % i for i in range(nl)] + ['g_log_var', 'g_pre'] + _STEM_NAMES)
    out['grads'] = _pairs([out.pop('_g%d' % i) for i in range(nl)])
    out['stem'] = tuple(out.pop(k) for k in _STEM_NAMES)
    return out


def value_rnn(stem, layers, x, h0, c0, ret, zs=None, masks=None):
    """RNN mode's value loss mean((v - ret)^2) over the B*L rows (ppo.py:311-353): ``grads`` per critic layer,
    ``stem`` as in ppo_policy_rnn, ``g_pre`` = dL/dv."""
    S = [f64(t).requires_grad_(True) for t in stem]
    L = _leaves(layers)
    v = trunk(_rnn_features(S, x, h0, c0, zs), L, masks=masks)
    ret = f64(ret).reshape(-1, 1).to(v.device)
    loss = (v - ret).pow(2).mean()
    st = {'loss': loss, 'explained_var': 1 - torch.var(ret - v) / torch.var(ret)}
    nl = 2 * len(L)
    out = _result(loss, st, _flat(L) + [v] + S, ['_g%d' % i for i in range(nl)] + ['g_pre'] + _STEM_NAMES)
    out['grads'] = _pairs([out.pop('_g%d' % i) for i in range(nl)])
    out['stem'] = tuple(out.pop(k) for k in _STEM_NAMES)
    return out


def ddpg_critic(layers, x, actions, y, aux_layer=1, weights=None):
    """nn.MSELoss()(Q(s, a), y) of oracle/ddpg.py: ``grads`` per critic layer, ``g_pre`` = dL/dQ, stats ``q_mean`` and
    ``q`` [B, 1].  ``weights`` [B] (prioritized replay's importance weights, dqn.py:148-168): mean(w (Q - y)^2)."""
    L = _leaves(layers)
    q = trunk(f64(x), L, aux=f64(actions), aux_layer=aux_layer)
    y = f64(y).reshape(-1, 1).to(q.device)
    if weights is None:
        loss = F.mse_loss(q, y)
    else:
        loss = (f64(weights).reshape(-1, 1).to(q.device) * (q - y).pow(2)).mean()
    out = _result(loss, {'loss': loss, 'q_mean': q.mean(), 'q': q}, _flat(L) + [q],
                  ['_g%d' % i for i in range(2 * len(L))] + ['g_pre'])
    out['grads'] = _pairs([out.pop('_g%d' % i) for i in range(2 * len(L))])
    return out


def ddpg_actor(actor, critic, x, aux_layer=1, actor_masks=None, critic_masks=None):
    """-mean Q(s, tanh(actor(s))) of oracle/ddpg.py through the critic's aux columns: ``grads`` per actor layer,
    ``g_action`` = dL/d(action) (what grad_wrt_aux computes), ``g_pre`` = dL/d(actor pre-tanh output)."""
    La, Lc = _leaves(actor), [(f64(w), f64(b)) for w, b in critic]
    pre = trunk(f64(x), La, masks=actor_masks)
    act = torch.tanh(pre)
    q = trunk(f64(x), Lc, aux=act, aux_layer=aux_layer, masks=critic_masks)
    loss = -q.mean()
    out = _result(loss, {'loss': loss}, _flat(La) + [pre, act],
                  ['_g%d' % i for i in range(2 * len(La))] + ['g_pre', 'g_action'])
    out['grads'] = _pairs([out.pop('_g%d' % i) for i in range(2 * len(La))])
    return out

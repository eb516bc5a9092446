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


def ppo_policy(layers, log_var, x, actions, adv, behave, mode, **hyper):
    """One policy update's loss on the actor ``layers`` over (already whitened) inputs ``x``: ``grads`` per layer,
    ``g_log_var``, ``g_pre``, plus the loss statistics."""
    L = _leaves(layers)
    lv = f64(log_var).reshape(-1).requires_grad_(True)
    pre = trunk(f64(x), L)
    ref = hyper.pop('ref', None)
    loss, st = _policy_loss(pre, lv, f64(actions), f64(adv), f64(behave), mode,
                            ref=f64(ref) if ref is not None else None, **hyper)
    out = _result(loss, st, _flat(L) + [lv, pre], ['_g%d' % i for i in range(2 * len(L))] + ['g_log_var', 'g_pre'])
    out['grads'] = _pairs([out.pop('_g%d' % i) for i in range(2 * len(L))])
    return out


def value(layers, x, ret):
    """_value_update's loss mean((v - ret)^2) and explained variance; ``grads`` per layer, ``g_pre`` = dL/dv."""
    L = _leaves(layers)
    v = trunk(f64(x), L)
    ret = f64(ret).reshape(-1, 1)
    loss = (v - ret).pow(2).mean()
    st = {'loss': loss, 'explained_var': 1 - torch.var(ret - v) / torch.var(ret), 'ret_mean': ret.mean()}
    out = _result(loss, st, _flat(L) + [v], ['_g%d' % i for i in range(2 * len(L))] + ['g_pre'])
    out['grads'] = _pairs([out.pop('_g%d' % i) for i in range(2 * len(L))])
    return out


def ddpg_critic(layers, x, actions, y, aux_layer=1):
    """nn.MSELoss()(Q(s, a), y) of oracle/ddpg.py: ``grads`` per critic layer, ``g_pre`` = dL/dQ, stat ``q_mean``."""
    L = _leaves(layers)
    q = trunk(f64(x), L, aux=f64(actions), aux_layer=aux_layer)
    loss = F.mse_loss(q, f64(y).reshape(-1, 1))
    out = _result(loss, {'loss': loss, 'q_mean': q.mean()}, _flat(L) + [q],
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

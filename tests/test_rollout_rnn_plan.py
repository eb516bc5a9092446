"""Host side of the recurrent persistent rollout (csrc/rollout_rnn.cu): which shapes `sb200_ppo_rollout_rnn_supported`
takes -- decided from the shapes alone, so no GPU is needed -- and each limit pinned on both sides.  Declined shapes run on
the per-step launch chain."""
import ctypes as C
import os
import re

import pytest

from surreal_b200 import _lib, ops

MAX_RNN_LAYERS = _lib.MAX_RNN_LAYERS


def _mlp(dims, acts=None, ln=False, aux=-1):
    m = _lib.Mlp()
    m.n_layers = len(dims) - 1
    for i, v in enumerate(dims):
        m.dims[i] = v
    for l in range(m.n_layers):
        m.act[l] = (acts[l] if acts is not None else (ops.ACT_TANH if l < m.n_layers - 1 else ops.ACT_NONE))
        m.ldw[l] = (dims[l + 1] + 3) // 4 * 4
    m.aux_layer, m.aux_dim = aux, 0
    if ln:
        m.ln_g[0] = m.ln_b[0] = 16                   # any non-NULL gain / bias marks LayerNorm after layer 0
    return m


def _supported(D=64, H=100, layers=1, head=(300, 200), A=8, head_ln=False, ih_ln=False, ih_act=None, ih_out=None,
               ih_in=None, aux=-1):
    base = _lib.PPORollout()
    net = _mlp([H] + list(head) + [A], ln=head_ln, aux=aux)
    base.net = C.pointer(net)
    base.N, base.D, base.A, base.T = 1024, D, A, 32
    r = _lib.PPORolloutRnn()
    r.base = C.pointer(base)
    ihs = [_mlp([(ih_in or D) if k == 0 else H, ih_out or 4 * H], acts=[ih_act or ops.ACT_NONE], ln=ih_ln)
           for k in range(min(layers, MAX_RNN_LAYERS))]
    for k, m in enumerate(ihs):
        r.ih[k] = C.pointer(m)
    r.layers, r.H = layers, H
    return _lib.lib().sb200_ppo_rollout_rnn_supported(C.byref(r)) == 1


def test_default_policy_is_taken():
    """The reference's default PPO policy (LSTM(100), head 300-200) at 1 and 2 layers; widths that are not multiples of 16."""
    assert _supported()
    assert _supported(layers=2)
    assert _supported(D=11, H=37, head=(30, 20), A=3, layers=2)
    assert _supported(D=1, H=1, head=(), A=1)


@pytest.mark.parametrize('field,ok,over', [
    ('layers', MAX_RNN_LAYERS, MAX_RNN_LAYERS + 1),
    ('H', 128, 129),
    ('D', 256, 257),
    ('A', 32, 33),
])
def test_plan_limits(field, ok, over):
    """Each limit on both sides: layers (SB200_MAX_RNN_LAYERS), H (one thread per gate column), the env's observation
    width and the action width (one warp lane per action dim)."""
    assert _supported(**{field: ok})
    assert not _supported(**{field: over})
    assert not _supported(**{field: 0})


def test_head_limits():
    """Head layers up to 512 wide, 1 .. SB200_MAX_LAYERS of them."""
    assert _supported(head=(512, 512))
    assert not _supported(head=(513, 200))
    assert not _supported(head=(300, 513))
    assert _supported(head=(64, 64, 64))                    # SB200_MAX_LAYERS = 4 layers


def test_declined_descriptors():
    """LayerNorm anywhere, an aux input, an input projection that is not one plain Linear in -> 4H, or an input width
    other than the env's observation (a CNN stem's features) take the per-step chain."""
    assert not _supported(head_ln=True)
    assert not _supported(ih_ln=True)
    assert not _supported(aux=1)
    assert not _supported(ih_act=ops.ACT_TANH)
    assert not _supported(ih_out=4 * 100 + 4)
    assert not _supported(ih_in=65)


def test_ctypes_structure_matches_the_header():
    """PPORolloutRnn has the fields of sb200_ppo_rollout_rnn, in order."""
    txt = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'surreal_b200.h')).read()
    txt = re.sub(r'/\*.*?\*/', '', txt, flags=re.S)
    body = re.search(r'typedef\s+struct\s+sb200_ppo_rollout_rnn\s*\{(.*?)\}\s*sb200_ppo_rollout_rnn\s*;', txt, re.S).group(1)
    names = []
    for decl in filter(None, (d.strip() for d in body.split(';'))):
        for d in re.match(r'(?:const\s+)?\w+\s*(.*)$', decl, re.S).group(1).split(','):
            names.append(re.match(r'[\s*]*(\w+)', d).group(1))
    assert [f[0] for f in _lib.PPORolloutRnn._fields_] == names

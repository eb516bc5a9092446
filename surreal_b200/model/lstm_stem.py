"""LSTM stem of RNN-mode PPO -- host-side mirror of the ``nn.LSTM(rnn_insize, rnn_hidden, rnn_layer, batch_first=True)`` the
reference's PPOModel puts in front of actor and critic (surreal/model/ppo_net.py:143-152,277-279,342-351; the DEFAULT PPO
config, ppo_configs.py:57-62), at any depth ``layers`` = rnn_layer (dropout 0, as the reference builds it).

Parameters live in ONE flat buffer as 2 * layers FlatNet segments in the order ih_0, hh_0, ih_1, hh_1, ... -- W_ih^T
[in][4H] + b_ih and W_hh^T [H][4H] + b_hh per layer, in = D for layer 0 and H above -- so the input projections and all
weight gradients are ordinary MLP-kernel calls, and each of the two optimisers that train the shared stem
(ppo_net.py:202-224) keeps its own flat Adam state over every layer.  At one layer the offsets are those of the
one-layer stem.  The recurrence itself is csrc/lstm.cu.

Layer 0 reads the z-filtered observation rows; layer l > 0 reads layer l-1's h_t (torch's stacking); every layer starts
from its own initial cells; the heads read the top layer's output.  Initial cells are passed per layer: None (zeros), a
list of per-layer [B, >= H] tensors whose row b starts at element b * ld_cells, or -- as torch holds them -- one
[layers, B, H] tensor (a single [B, H] tensor at one layer)."""
import ctypes as C

import torch

from .. import _lib, ops
from .._lib import check
from ..ops import _ptr


def _sfx(k):
    return '' if k == 0 else str(k)


class LSTMStem:
    def __init__(self, in_dim, hidden, device, layers=1):
        assert int(layers) >= 1, 'rnn_layer must be at least 1'
        assert 4 * hidden <= 1024, 'rnn_hidden up to 256'
        self.D, self.H, self.layers = int(in_dim), int(hidden), int(layers)
        self.device = torch.device(device)
        self.ihs = [ops.FlatNet([self.D if k == 0 else self.H, 4 * self.H], [ops.ACT_NONE], self.device) for k in range(self.layers)]
        self.hhs = [ops.FlatNet([self.H, 4 * self.H], [ops.ACT_NONE], self.device) for k in range(self.layers)]
        self.ih, self.hh = self.ihs[0], self.hhs[0]
        self.off, o = {}, 0
        for k in range(self.layers):
            for name, net in (('ih', self.ihs[k]), ('hh', self.hhs[k])):
                self.off[name + _sfx(k)] = (o, net.size)
                o += net.size
        self.size = o
        self.params = torch.zeros(self.size, dtype=torch.float32, device=self.device)
        for k in range(self.layers):
            self.ihs[k].params, self.hhs[k].params = self.seg('ih' + _sfx(k)), self.seg('hh' + _sfx(k))
        ref = torch.nn.LSTM(self.D, self.H, self.layers, batch_first=True)   # torch's default initialisation
        self.load_torch({k: v.detach() for k, v in ref.state_dict().items()})

    def seg(self, name, buf=None):
        """Segment ``name`` ('ih' / 'hh' for layer 0, 'ih<k>' / 'hh<k>' for layer k) of the flat buffer."""
        o, n = self.off[name]
        return (self.params if buf is None else buf)[o:o + n]

    def load_torch(self, sd, prefix=''):
        f = lambda k: torch.as_tensor(sd[prefix + k], dtype=torch.float32)  # noqa: E731
        for k in range(self.layers):
            self.ihs[k].set_layer(0, f('weight_ih_l%d' % k), f('bias_ih_l%d' % k))
            self.hhs[k].set_layer(0, f('weight_hh_l%d' % k), f('bias_hh_l%d' % k))

    def state_items(self, prefix='rnn_stem.'):
        items = []
        for k in range(self.layers):
            wi, bi = self.ihs[k].get_layer(0)
            wh, bh = self.hhs[k].get_layer(0)
            items += [(prefix + 'weight_ih_l%d' % k, wi), (prefix + 'weight_hh_l%d' % k, wh),
                      (prefix + 'bias_ih_l%d' % k, bi), (prefix + 'bias_hh_l%d' % k, bh)]
        return items

    def buffers(self, B, L, save=True):
        """Work buffers of B sequences x L steps.  pre_x is shared by the layers.  With ``save`` every layer k keeps its
        own h_out / h_prev / gates / c_seq (keys suffixed with k for k > 0) for the backward pass; without, the layers
        take turns on two h_out buffers and the top layer always writes 'h_out'."""
        f = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        H, R = self.H, B * L
        Hp = ops._ru(H, 4)                                        # row stride of the h buffers (16-byte rows for the GEMM kernels)
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        b = dict(pre_x=f(R, 4 * H))
        if save:
            for k in range(self.layers):
                s = _sfx(k)
                b.update({'h_out' + s: z(R, Hp)[:, :H], 'h_prev' + s: z(R, Hp)[:, :H], 'gates' + s: f(R, 4 * H), 'c_seq' + s: f(R, H)})
        else:
            b['h_out'] = z(R, Hp)[:, :H]
            if self.layers > 1:
                b['h_out1'] = z(R, Hp)[:, :H]
        return b

    def layer_bufs(self, bufs, k):
        """Layer k's buffers out of ``buffers()``: h_out (and, saved, h_prev / gates / c_seq)."""
        if 'gates' in bufs:
            s = _sfx(k)
            return {name: bufs.get(name + s) for name in ('h_out', 'h_prev', 'gates', 'c_seq')}
        return {'h_out': bufs['h_out' if (self.layers - 1 - k) % 2 == 0 else 'h_out1']}

    def per_layer(self, cells):
        """Initial / last cells as a list with one entry per layer (see the module docstring)."""
        if cells is None:
            return [None] * self.layers
        if isinstance(cells, torch.Tensor):
            if self.layers == 1:
                return [cells]
            assert cells.dim() == 3 and cells.shape[0] == self.layers, 'cells of a %d-layer stem: [layers, B, H]' % self.layers
            return list(cells.unbind(0))
        cells = list(cells)
        assert len(cells) == self.layers, 'cells for %d layers, got %d' % (self.layers, len(cells))
        return cells

    def forward(self, xf, h0, c0, ld_cells, B, L, bufs, h_last=None, c_last=None, params=None):
        """xf: [B*L, D] (already z-filtered, sequence-major rows b*L + t); h0 / c0: initial cells per layer (see the module
        docstring), row b of each at element b*ld_cells; h_last / c_last: per-layer [B, H] outputs (may be h0 / c0 for an
        in-place update).  -> the top layer's h_out [B*L, H]."""
        P = self.params if params is None else params
        h0, c0, h_last, c_last = self.per_layer(h0), self.per_layer(c0), self.per_layer(h_last), self.per_layer(c_last)
        x = xf
        for k in range(self.layers):
            lb = self.layer_bufs(bufs, k)
            ops.mlp_forward(self.ihs[k], x, params=self.seg('ih' + _sfx(k), P), out=bufs['pre_x'])
            lay = self.hhs[k].layout[0]
            hh = self.seg('hh' + _sfx(k), P)
            check(_lib.lib().sb200_lstm_forward_f32(
                _ptr(bufs['pre_x']), C.c_void_p(hh.data_ptr() + 4 * lay['w']), C.c_void_p(hh.data_ptr() + 4 * lay['b']), _ptr(h0[k]),
                _ptr(c0[k]), int(ld_cells), B, L, self.H, lb['h_out'].stride(0), _ptr(lb['h_out']), _ptr(lb.get('h_prev')),
                _ptr(lb.get('gates')), _ptr(lb.get('c_seq')), _ptr(h_last[k]), _ptr(c_last[k]), ops._stream()), 'sb200_lstm_forward_f32')
            x = lb['h_out']
        return x


class RnnTrainer:
    """Saved activations, BPTT and gradient slabs of the LSTM stem for ONE optimiser on B sequences of L steps."""

    def __init__(self, stem, B, L, splits=None):
        self.stem, self.B, self.L = stem, B, L
        dev = stem.device
        R = B * L
        self.splits = splits if splits is not None else max(1, min(16, R // 128))
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)  # noqa: E731
        self.bufs = stem.buffers(B, L, save=True)
        self.slabs = z(self.splits, stem.size)
        self.exp_avg, self.exp_avg_sq = z(stem.size), z(stem.size)
        self.dpres = [z(R, 4 * stem.H) for _ in range(stem.layers)]     # per layer: gradient w.r.t. the gate pre-activations
        self.dpre = self.dpres[0]
        # gradient w.r.t. the outputs of layers 0 .. layers-2, from the input projection of the layer above
        self.dh = [z(R, ops._ru(stem.H, 4)) for _ in range(stem.layers - 1)]
        self.xf = self.h0 = self.c0 = None
        self.ld_cells = 0

    def forward(self, xf, h0, c0, ld_cells):
        self.xf, self.h0, self.c0, self.ld_cells = xf, h0, c0, ld_cells
        return self.stem.forward(xf, h0, c0, ld_cells, self.B, self.L, self.bufs)

    def backward(self, dh_out):
        """dh_out [B*L, >= H]: gradient w.r.t. the top layer's outputs (the head's input gradient, no activation in
        between).  BPTT from the top layer down; each layer's input projection hands the layer below its output gradient."""
        s, L_, st = self.stem, _lib.lib(), ops._stream()
        R, G = self.B * self.L, 4 * s.H
        c0 = s.per_layer(self.c0)
        base = self.slabs.data_ptr()
        dh = dh_out
        for k in reversed(range(s.layers)):
            lb, dpre = s.layer_bufs(self.bufs, k), self.dpres[k]
            ih, hh = s.ihs[k], s.hhs[k]
            lay_h, lay_i = hh.layout[0], ih.layout[0]
            check(L_.sb200_lstm_backward_f32(_ptr(dh), dh.stride(0), _ptr(lb['gates']), _ptr(lb['c_seq']), _ptr(c0[k]), int(self.ld_cells),
                                             C.c_void_p(hh.params.data_ptr() + 4 * lay_h['w']), self.B, self.L, s.H, _ptr(dpre), st),
                  'sb200_lstm_backward_f32')
            X = self.xf if k == 0 else s.layer_bufs(self.bufs, k - 1)['h_out']
            o_ih, o_hh = s.off['ih' + _sfx(k)][0], s.off['hh' + _sfx(k)][0]
            check(L_.sb200_linear_bwd_dw_f32(_ptr(X), X.stride(0), _ptr(dpre), G, C.c_void_p(base + 4 * (o_ih + lay_i['w'])),
                                             C.c_void_p(base + 4 * (o_ih + lay_i['b'])), s.size, self.splits, lay_i['ldw'], R,
                                             ih.dims[0], G, st), 'sb200_linear_bwd_dw_f32(lstm ih)')
            hp = lb['h_prev']
            check(L_.sb200_linear_bwd_dw_f32(_ptr(hp), hp.stride(0), _ptr(dpre), G, C.c_void_p(base + 4 * (o_hh + lay_h['w'])),
                                             C.c_void_p(base + 4 * (o_hh + lay_h['b'])), s.size, self.splits, lay_h['ldw'], R, s.H, G, st),
                  'sb200_linear_bwd_dw_f32(lstm hh)')
            if k > 0:                                             # dh_out of layer k-1 = dpre_k . W_ih_k (no activation)
                dh = self.dh[k - 1]
                check(L_.sb200_linear_bwd_dx_f32(_ptr(dpre), G, C.c_void_p(ih.params.data_ptr() + 4 * lay_i['w']), lay_i['ldw'], None, 0,
                                                 _ptr(dh), dh.stride(0), R, G, s.H, st), 'sb200_linear_bwd_dx_f32(lstm layer input)')

    def backward_input(self, dx, x_act):
        """After ``backward``: the gradient w.r.t. layer 0's input, dpre_0 . W_ih_0, masked by relu'(x_act) -- i.e. w.r.t.
        the pre-activation of a ReLU layer in front of the stem whose output ``x_act`` [B*L, D] the stem read (the CNN
        stem's features) -- into ``dx`` [B*L, >= D]."""
        s, R, G = self.stem, self.B * self.L, 4 * self.stem.H
        ih, lay = s.ihs[0], s.ihs[0].layout[0]
        check(_lib.lib().sb200_linear_bwd_dx_f32(_ptr(self.dpres[0]), G, C.c_void_p(ih.params.data_ptr() + 4 * lay['w']), lay['ldw'],
                                                 _ptr(x_act), x_act.stride(0), _ptr(dx), dx.stride(0), R, G, s.D, ops._stream()),
              'sb200_linear_bwd_dx_f32(lstm stem input)')

    def state_dict(self):
        return {'exp_avg': self.exp_avg.detach().clone(), 'exp_avg_sq': self.exp_avg_sq.detach().clone()}

    def load_state_dict(self, sd):
        self.exp_avg.copy_(torch.as_tensor(sd['exp_avg']).to(self.stem.device))
        self.exp_avg_sq.copy_(torch.as_tensor(sd['exp_avg_sq']).to(self.stem.device))


def rows_zfilter(x, row_stride, batch_stride, B, L, D, zf_stats, zf_eps, out):
    """out[b*L + t, :D] = zfilter(x[b*batch_stride + t*row_stride : +D]) (plain gather when zf_stats is None)."""
    check(_lib.lib().sb200_rows_zfilter_f32(_ptr(x), int(row_stride), int(batch_stride), B, L, D, _ptr(zf_stats), float(zf_eps), _ptr(out),
                                            out.stride(0), ops._stream()), 'sb200_rows_zfilter_f32')
    return out

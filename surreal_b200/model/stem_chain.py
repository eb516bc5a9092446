"""The stems a PPO learner runs between a batch record row and its heads' input: PPOModel.stems, i.e. [cnn], [lstm] or
[cnn, lstm] (frames through the CNN stem, its features through the LSTM stem).  They are shared by actor and critic and
trained by BOTH optimisers (ppo_net.py:202-224), each with its own Adam state.  An empty list is MLP mode, where the heads
z-filter the observation rows themselves and none of this runs."""
import torch

from .. import ops
from .cnn_stem import StemTrainer, joint_step
from .lstm_stem import RnnTrainer, rows_zfilter


class StemChain:
    """One learner's stem path: the gathered input rows, the inference buffers of the critic pass (B*(n+1) rows) and of
    the reference model (B*E update rows); each optimiser trains the stems through its own ChainTrainer.

    Input rows are gathered from the records [B, n+1, ld] with rows_zfilter: the model's z-filtered observation for an
    LSTM-first chain, the raw frame words (a float load / store copies the bits of any word, denormal and NaN patterns too)
    for a CNN-first chain.  A CNN-only critic pass reads the frames in place: its records hold nothing but the frame."""

    def __init__(self, model, ref_model, obs_full, E):
        self.model, self.ref_model = model, ref_model
        self.cnn, self.rnn = model.cnn_stem, model.rnn_stem
        B, n1, ld = obs_full.shape
        self.obs_full, self.B, self.n1, self.E, self.M = obs_full, B, n1, E, B * E
        self.od = self.cnn.C * self.cnn.H * self.cnn.W // 4 if self.cnn is not None else model.low_dim
        self.size = sum(s.size for s in model.stems)
        # the heads' input gradient: as is behind the LSTM's output, times relu'(features) behind the CNN's Linear + ReLU
        self.input_grad = 'linear' if self.rnn is not None else 'relu'
        dev = obs_full.device
        zz = lambda r: torch.zeros(r, ops._ru(self.od, 4), dtype=torch.float32, device=dev)[:, :self.od]  # noqa: E731
        self.x_eff = zz(self.M)
        self.x_all = zz(B * n1) if self.rnn is not None else obs_full.view(B * n1, ld)
        # the reference model's update rows through its own z-filter; frames need no filter
        self.x_ref = zz(self.M) if self.cnn is None else self.x_eff
        self.bufs_all = self._bufs(model, B * n1, n1)
        self.bufs_ref = self._bufs(ref_model, self.M, E)

    def _bufs(self, model, rows, L):
        return dict(cnn=model.cnn_stem.buffers(rows) if model.cnn_stem is not None else None,
                    rnn=model.rnn_stem.buffers(self.B, L, save=False) if model.rnn_stem is not None else None)

    def frames(self, rows):
        """Frame rows [R, od words] as the uint8 [R, C, H, W] frames the CNN stem reads."""
        return rows.view(torch.uint8).view(rows.shape[0], self.cnn.C, self.cnn.H, self.cnn.W)

    def gather(self):
        """Once per learn(): the update rows (the first E steps of every window), and with an LSTM the critic pass's rows
        and the reference model's update rows (ppo.py:507-539)."""
        m, ref, B, n1, o = self.model, self.ref_model, self.B, self.n1, self.obs_full
        ld = o.shape[2]
        if self.rnn is not None:
            rows_zfilter(o, ld, n1 * ld, B, n1, self.od, m.z_stats, m.z_eps, self.x_all)
        rows_zfilter(o, ld, n1 * ld, B, self.E, self.od, m.z_stats, m.z_eps, self.x_eff)
        if self.x_ref is not self.x_eff:
            rows_zfilter(o, ld, n1 * ld, B, self.E, self.od, ref.z_stats, ref.z_eps, self.x_ref)

    def _forward(self, model, x, cells, L, bufs):
        if model.cnn_stem is not None:
            x = model.cnn_stem.forward(self.frames(x), bufs['cnn'])
        if model.rnn_stem is not None:
            x = model.rnn_stem.forward(x, *cells, self.B, L, bufs['rnn'])
        return x

    def critic_features(self, cells):
        """The heads' input on all B*(n+1) rows (the LSTM from the windows' initial ``cells`` (h0, c0, ld))."""
        return self._forward(self.model, self.x_all, cells, self.n1, self.bufs_all)

    def ref_features(self, cells):
        """The reference model's heads' input on the B*E update rows."""
        return self._forward(self.ref_model, self.x_ref, cells, self.E, self.bufs_ref)


class ChainTrainer:
    """The stems' trainers of ONE optimiser whose head is ``head`` (ops.MlpTrainer): ``cnn`` (StemTrainer) and ``rnn``
    (RnnTrainer), None where the chain has no such stem, and the joint gradient [head | CNN | LSTM] the optimiser steps;
    ``head.grad`` is its head segment."""

    def __init__(self, chain, head):
        self.chain, self.head = chain, head
        self.cnn = StemTrainer(chain.cnn, chain.M) if chain.cnn is not None else None
        self.rnn = RnnTrainer(chain.rnn, chain.B, chain.E) if chain.rnn is not None else None
        self.stems = [t for t in (self.cnn, self.rnn) if t is not None]
        nh = head.net.size
        self.grad = torch.zeros(nh + chain.size, dtype=torch.float32, device=chain.obs_full.device)
        head.grad = self.grad[:nh]

    def forward(self, cells):
        """Training forward on the update rows -> the head's input [B*E, width]."""
        x = self.chain.x_eff
        if self.cnn is not None:
            x = self.cnn.forward(self.chain.frames(x))
        if self.rnn is not None:
            x = self.rnn.forward(x, *cells)
        return x

    def step(self, norm_out, stop_flag=None):
        """After the head's backward: the stems' backward from the head's input gradient, in reverse (the LSTM hands the
        CNN its input gradient masked by relu'(features)), then ONE joint step over [head | CNN | LSTM]."""
        d = self.head.dx0
        if self.rnn is not None:
            self.rnn.backward(d)
            if self.cnn is not None:
                self.rnn.backward_input(self.cnn.d_fc, self.cnn.bufs['feat'])
                d = self.cnn.d_fc
        if self.cnn is not None:
            self.cnn.backward(d)
        joint_step(self.head, self.stems, self.grad, norm_out=norm_out, stop_flag=stop_flag)

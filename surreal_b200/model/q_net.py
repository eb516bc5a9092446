"""Q network of DQN as flat device buffers (host-side mirror of surreal/model/q_net.py:9-65,122-134: DuelingQbase and
build_ffqfunc).  The action tower Linear-ReLU-...-Linear(n_actions) is one FlatNet; with ``dueling`` the state tower over
the same hidden sizes ending in Linear(1) is a second FlatNet reading the same input, and Q = (A - mean_j A) + V is formed
by the act / TD kernels (csrc/dqn.cu).  The pixel path (``convs``) is not built."""
import collections

import torch

from .. import ops
from .ppo_net import _default_linear_init


class QModel:
    def __init__(self, obs_spec, action_dim, fc_hidden_sizes, dueling, convs=None, device=None):
        self.device = torch.device(device if device is not None else 'cuda')
        if self.device.type != 'cuda':
            raise RuntimeError('surreal_b200 has no CPU path: QModel needs a CUDA device')
        if convs or 'pixel' in obs_spec:
            raise NotImplementedError('the convolutional Q function (q_net.py:68-119) is not built: model.convs must be '
                                      'empty and the observations low-dimensional')
        self.action_dim = int(action_dim)
        self.dueling = bool(dueling)
        self.input_dim = obs_spec['low_dim']['flat_inputs'][0]
        D, h = self.input_dim, list(fc_hidden_sizes)
        R, N = ops.ACT_RELU, ops.ACT_NONE
        self.action_net = ops.FlatNet([D] + h + [self.action_dim], [R] * len(h) + [N], self.device)
        self.action_net.load_layers(_default_linear_init(self.action_net.dims))
        self.state_net = None
        if self.dueling:
            self.state_net = ops.FlatNet([D] + h + [1], [R] * len(h) + [N], self.device)
            self.state_net.load_layers(_default_linear_init(self.state_net.dims))

    def nets(self):
        """[action tower] or [action tower, state tower]."""
        return [self.action_net] + ([self.state_net] if self.dueling else [])

    def flat_state(self):
        st = {'action': self.action_net.params}
        if self.dueling:
            st['state'] = self.state_net.params
        return st

    def load_flat_state(self, st):
        self.action_net.params.copy_(st['action'])
        if self.dueling:
            self.state_net.params.copy_(st['state'])

    def copy_from(self, other):
        for a, b in zip(self.nets(), other.nets()):
            a.params.copy_(b.params)

    def _keys(self):
        out = [(self.action_net, l, 'fc_action_layers.%d' % l) for l in range(self.action_net.n_layers)]
        if self.dueling:
            out += [(self.state_net, l, 'fc_state_layers.%d' % l) for l in range(self.state_net.n_layers)]
        return out

    def state_dict(self):
        """The reference's keys: fc_action_layers.{i}.{weight,bias} (and fc_state_layers.{i}.* with dueling)."""
        sd = collections.OrderedDict()
        for net, l, key in self._keys():
            sd[key + '.weight'], sd[key + '.bias'] = net.get_layer(l)
        return sd

    def load_state_dict(self, sd):
        for net, l, key in self._keys():
            net.set_layer(l, torch.as_tensor(sd[key + '.weight'], dtype=torch.float32),
                          torch.as_tensor(sd[key + '.bias'], dtype=torch.float32))

    def forward_towers(self, obs, adv_out=None, value_out=None):
        """(action tower output [rows, n_actions], state tower output [rows, 1] or None) on the fused forward."""
        a = ops.mlp_forward(self.action_net, obs, out=adv_out)
        v = ops.mlp_forward(self.state_net, obs, out=value_out) if self.dueling else None
        return a, v

"""DDPG actor / critic as flat device buffers (host-side mirror of surreal/model/ddpg_net.py:13-95 and
builders.py:35-84).  The critic's cat(h, action) before its second layer (builders.py:80-83) is the fused
forward kernel's ``aux_layer = 1``: no concatenated tensor is materialised.  With ``use_layernorm`` every hidden layer is
Linear -> ReLU -> LayerNorm (builders.py:42-48,64-77), the critic's action joining after the first LayerNorm."""
import collections

import torch

from .. import ops
from .ppo_net import _default_linear_init


class DDPGModel:
    def __init__(self, obs_spec, action_dim, use_layernorm, actor_fc_hidden_sizes, critic_fc_hidden_sizes,
                 conv_out_channels=None, conv_kernel_sizes=None, conv_strides=None, conv_hidden_dim=None,
                 critic_only=False, device=None):
        self.device = torch.device(device if device is not None else 'cuda')
        if self.device.type != 'cuda':
            raise RuntimeError('surreal_b200 has no CPU path: DDPGModel needs a CUDA device')
        self.is_pixel_input = 'pixel' in obs_spec
        if self.is_pixel_input:
            raise NotImplementedError('CNN perception stem (builders.py:8-33) is not built yet (SURVEY §8 K16)')
        self.action_dim = action_dim
        self.use_layernorm = bool(use_layernorm)
        self.input_dim = obs_spec['low_dim']['flat_inputs'][0]
        D, A = self.input_dim, action_dim
        R, T, N = ops.ACT_RELU, ops.ACT_TANH, ops.ACT_NONE
        ah, ch = list(actor_fc_hidden_sizes), list(critic_fc_hidden_sizes)
        ln = self.use_layernorm
        self.actor = None
        if not critic_only:
            self.actor = ops.FlatNet([D] + ah + [A], [R] * len(ah) + [T], self.device, layernorm=ln)
            self.actor.load_layers(_default_linear_init(self.actor.dims))
        self.critic = ops.FlatNet([D] + ch + [1], [R] * len(ch) + [N], self.device, aux_layer=1, aux_dim=A, layernorm=ln)
        cd = [D, ch[0]]
        layers = _default_linear_init(cd) + _default_linear_init([ch[0] + A] + ch[1:] + [1])
        self.critic.load_layers(layers)

    def flat_state(self):
        st = {'critic': self.critic.params}
        if self.actor is not None:
            st['actor'] = self.actor.params
        return st

    def load_flat_state(self, st):
        self.critic.params.copy_(st['critic'])
        if self.actor is not None and 'actor' in st:
            self.actor.params.copy_(st['actor'])

    # state-dict keys: a Sequential index per layer (Linear, ReLU[, LayerNorm]) as the reference's Functional numbers them
    def _keys(self):
        """[(net, layer, linear key prefix, LayerNorm key prefix or None)] in the reference's state-dict order."""
        step = 3 if self.use_layernorm else 2
        ln = lambda pre, i: ('%s%d' % (pre, i + 2)) if self.use_layernorm else None  # noqa: E731
        out = []
        if self.actor is not None:
            for l in range(self.actor.n_layers):
                pre = 'actor.model.seq.'
                out.append((self.actor, l, '%s%d' % (pre, step * l),
                            ln(pre, step * l) if l + 1 < self.actor.n_layers else None))
        out.append((self.critic, 0, 'critic.model_obs.seq.0', ln('critic.model_obs.seq.', 0)))
        for l in range(1, self.critic.n_layers):
            pre = 'critic.model_concat.seq.'
            out.append((self.critic, l, '%s%d' % (pre, step * (l - 1)),
                        ln(pre, step * (l - 1)) if l + 1 < self.critic.n_layers else None))
        return out

    def state_dict(self):
        sd = collections.OrderedDict()
        for net, l, key, ln_key in self._keys():
            sd[key + '.weight'], sd[key + '.bias'] = net.get_layer(l)
            if ln_key is not None:
                sd[ln_key + '.weight'], sd[ln_key + '.bias'] = net.get_ln(l)
        return sd

    def load_state_dict(self, sd):
        g = lambda k: torch.as_tensor(sd[k], dtype=torch.float32)  # noqa: E731
        for net, l, key, ln_key in self._keys():
            net.set_layer(l, g(key + '.weight'), g(key + '.bias'))
            if ln_key is not None:
                net.set_ln(l, g(ln_key + '.weight'), g(ln_key + '.bias'))

    def forward_actor(self, obs):
        return ops.mlp_forward(self.actor, obs)

    def forward_critic(self, obs, action):
        return ops.mlp_forward(self.critic, obs, aux=action)

    def forward_perception(self, obs):
        return obs['low_dim']['flat_inputs'] if isinstance(obs, dict) else obs

    def forward(self, obs_in, calculate_value=True, action=None):
        x = self.forward_perception(obs_in)
        if action is None:
            action = self.forward_actor(x)
        value = self.forward_critic(x, action) if calculate_value else None
        return action, value

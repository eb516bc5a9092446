"""PPO actor / critic / z-filter as flat device buffers (host-side mirror of surreal/model/ppo_net.py:94-375,
model_builders/builders.py:86-175, z_filter.py:7-107).  Every forward is one fused CUDA launch."""
import collections

import torch

from .. import _lib, ops


class DiagGauss:
    """Shape bookkeeping only; the distribution math runs inside the loss kernels (csrc/ppo_loss.cu)."""
    pd_type = _lib.PD_GAUSSIAN

    def __init__(self, action_dim):
        self.d = action_dim


class Categorical:
    """Categorical policy of a discrete action space over ``n_actions`` logits (tests/cat_ref.py): pd rows
    [p | log p], one-hot action rows.  Shape bookkeeping only; the math runs in csrc/ppo_cat.cu."""
    pd_type = _lib.PD_CATEGORICAL

    def __init__(self, n_actions):
        self.d = n_actions


def make_pd(action_spec):
    """The policy distribution of an action_spec: Categorical for {'type': 'discrete', 'dim': (K,)}, 2 <= K <=
    SB200_PPO_CAT_MAX_K, else DiagGauss."""
    from ..session import ConfigError
    t = str(action_spec['type'] if isinstance(action_spec, dict) else action_spec.type)
    d = int((action_spec['dim'] if isinstance(action_spec, dict) else action_spec.dim)[0])
    if t == 'continuous':
        return DiagGauss(d)
    if t != 'discrete':
        raise ConfigError('action_spec.type must be "continuous" or "discrete", got %r' % t)
    if not 2 <= d <= _lib.PPO_CAT_MAX_K:
        raise ConfigError('a discrete action_spec needs 2 <= dim <= %d (the widest layer the fused forward accepts), '
                          'got %d' % (_lib.PPO_CAT_MAX_K, d))
    return Categorical(d)


def _default_linear_init(dims, seed_gen=None):
    """torch.nn.Linear's default initialisation (the un-vendored torchx L.Linear default is unknown,
    SURVEY §8c; parity tests always inject weights)."""
    layers = []
    for i in range(len(dims) - 1):
        lin = torch.nn.Linear(dims[i], dims[i + 1])
        layers.append((lin.weight.detach().clone(), lin.bias.detach().clone()))
    return layers


class PPOModel:
    """Same constructor keywords as the reference's PPOModel (ppo_net.py:110-118).  The LSTM stem (rnn_layer layers) is
    model/lstm_stem.py; the CNN stem (pixel input) is model/cnn_stem.py.  With both, frames run through the CNN stem,
    its features through the LSTM stem, and the heads read the LSTM's output."""

    def __init__(self, obs_spec, action_dim, model_config, use_cuda=True, init_log_sig=0, use_z_filter=False,
                 if_pixel_input=False, rnn_config=None, device=None, categorical=False):
        self.device = torch.device(device if device is not None else 'cuda')
        if self.device.type != 'cuda':
            raise RuntimeError('surreal_b200 has no CPU path: PPOModel needs a CUDA device')
        self.obs_spec, self.action_dim, self.model_config = obs_spec, action_dim, model_config
        self.use_z_filter, self.init_log_sig = use_z_filter, init_log_sig
        self.if_pixel_input, self.rnn_config = if_pixel_input, rnn_config
        # categorical: the actor head's last layer is linear with action_dim outputs (the logits) and there is no log_var
        self.categorical = bool(categorical)
        self.cnn_stem = None
        self.rnn_stem = None
        self.if_rnn = bool(rnn_config is not None and rnn_config.if_rnn_policy)
        self.low_dim = 0
        if 'low_dim' in obs_spec:
            for key in obs_spec['low_dim']:
                self.low_dim += obs_spec['low_dim'][key][0]
        if if_pixel_input:
            # optional CNN stem feature extractor (ppo_net.py:136-140), shared by actor and critic
            if self.low_dim > 0:
                raise NotImplementedError('mixed low_dim + pixel observations (ppo_net.py:268-275 concatenates them) are not '
                                          'supported: the HBM replay records carry one observation kind')
            from .cnn_stem import CNNStem
            self.cnn_stem = CNNStem(obs_spec['pixel']['camera0'], model_config.cnn_feature_dim, self.device)
        in_dim = self.low_dim + (model_config.cnn_feature_dim if if_pixel_input else 0)
        if self.if_rnn:
            # optional LSTM stem feature extractor (ppo_net.py:143-152), shared by actor and critic; with pixel input it
            # reads the CNN stem's features (the two stems in series, ppo_net.py:268-279)
            from .lstm_stem import LSTMStem
            if int(rnn_config.rnn_layer) < 1:
                from ..session import ConfigError
                raise ConfigError('algo.rnn.rnn_layer must be at least 1, got %d' % int(rnn_config.rnn_layer))
            self.rnn_stem = LSTMStem(in_dim, rnn_config.rnn_hidden, self.device, layers=rnn_config.rnn_layer)
            in_dim = rnn_config.rnn_hidden
        # the stems between an observation and the heads, in order: [], [cnn], [lstm] or [cnn, lstm]
        self.stems = [s for s in (self.cnn_stem, self.rnn_stem) if s is not None]
        D, A = in_dim, action_dim
        ah, ch = list(model_config.actor_fc_hidden_sizes), list(model_config.critic_fc_hidden_sizes)
        R, T, N = ops.ACT_RELU, ops.ACT_TANH, ops.ACT_NONE
        if self.categorical:
            self.actor = ops.FlatNet([D] + ah + [A], [R] * len(ah) + [N], self.device)
            self.actor.load_layers(_default_linear_init(self.actor.dims))
        else:
            self.actor = ops.FlatNet([D] + ah + [A], [R] * len(ah) + [T], self.device, extra=A)
            self.actor.load_layers(_default_linear_init(self.actor.dims), extra=torch.zeros(A) + init_log_sig)
        self.critic = ops.FlatNet([D] + ch + [1], [R] * len(ch) + [N], self.device)
        self.critic.load_layers(_default_linear_init(self.critic.dims))
        self.z_eps = 1e-5
        self.z_stats = None
        if use_z_filter:
            assert self.low_dim > 0, 'No low dimensional input, please turn off z-filter'
            self.z_stats = torch.cat([torch.zeros(self.low_dim), self.z_eps * torch.ones(self.low_dim),
                                      torch.tensor([self.z_eps])]).to(self.device)

    # -- parameters --------------------------------------------------------------------------------
    @property
    def log_var(self):
        """The Gaussian policy's log_var; None for the categorical policy."""
        return None if self.categorical else self.actor.extra_view()

    def update_target_params(self, net):
        """ppo_net.py:226-242: actor, critic and z-filter."""
        self.actor.params.copy_(net.actor.params)
        self.critic.params.copy_(net.critic.params)
        if self.cnn_stem is not None:
            self.cnn_stem.params.copy_(net.cnn_stem.params)
        if self.rnn_stem is not None:
            self.rnn_stem.params.copy_(net.rnn_stem.params)
        if self.use_z_filter:
            self.z_stats.copy_(net.z_stats)

    def update_target_z_filter(self, net):
        if self.use_z_filter:
            self.z_stats.copy_(net.z_stats)

    def flat_state(self):
        """The raw device buffers (kernel layout) -- what the collapsed parameter wire ships."""
        st = {'actor': self.actor.params, 'critic': self.critic.params}
        if self.cnn_stem is not None:
            st['cnn_stem'] = self.cnn_stem.params
        if self.rnn_stem is not None:
            st['rnn_stem'] = self.rnn_stem.params
        if self.use_z_filter:
            st['z_stats'] = self.z_stats
        return st

    def load_flat_state(self, st):
        self.actor.params.copy_(st['actor'])
        self.critic.params.copy_(st['critic'])
        if self.cnn_stem is not None and 'cnn_stem' in st:
            self.cnn_stem.params.copy_(st['cnn_stem'])
        if self.rnn_stem is not None and 'rnn_stem' in st:
            self.rnn_stem.params.copy_(st['rnn_stem'])
        if self.use_z_filter and 'z_stats' in st:
            self.z_stats.copy_(st['z_stats'])

    def state_dict(self):
        """Keys follow the reference module tree (actor.log_var, actor.model.*, critic.model.*, z_filter.*);
        Linear weights are exported in torch's [out, in] convention.  The categorical policy has no actor.log_var."""
        sd = collections.OrderedDict()
        if self.cnn_stem is not None:
            for k, v in self.cnn_stem.state_items():
                sd[k] = v
        if self.rnn_stem is not None:
            for k, v in self.rnn_stem.state_items():
                sd[k] = v
        if not self.categorical:
            sd['actor.log_var'] = self.log_var.detach().clone().view(1, -1)
        for name, net in (('actor', self.actor), ('critic', self.critic)):
            for l in range(net.n_layers):
                w, b = net.get_layer(l)
                sd['%s.model.seq.%d.weight' % (name, 2 * l)] = w
                sd['%s.model.seq.%d.bias' % (name, 2 * l)] = b
        if self.use_z_filter:
            D = self.low_dim
            sd['z_filter.running_sum'] = self.z_stats[:D].clone()
            sd['z_filter.running_sumsq'] = self.z_stats[D:2 * D].clone()
            sd['z_filter.count'] = self.z_stats[2 * D:].clone()
        return sd

    def load_state_dict(self, sd):
        g = lambda k: torch.as_tensor(sd[k], dtype=torch.float32)  # noqa: E731
        if ('actor.log_var' in sd) == self.categorical:
            have, want = ('Gaussian', 'categorical') if self.categorical else ('categorical', 'Gaussian')
            raise ValueError('state_dict holds a %s policy (%s actor.log_var) but this PPOModel has a %s policy'
                             % (have, 'with' if have == 'Gaussian' else 'without', want))
        if self.cnn_stem is not None:
            self.cnn_stem.load_state(sd)
        if self.rnn_stem is not None:
            self.rnn_stem.load_torch(sd, prefix='rnn_stem.')
        if not self.categorical:
            self.log_var.copy_(g('actor.log_var').reshape(-1).to(self.device))
        for name, net in (('actor', self.actor), ('critic', self.critic)):
            for l in range(net.n_layers):
                net.set_layer(l, g('%s.model.seq.%d.weight' % (name, 2 * l)), g('%s.model.seq.%d.bias' % (name, 2 * l)))
        if self.use_z_filter and 'z_filter.count' in sd:
            self.z_stats.copy_(torch.cat([g('z_filter.running_sum').reshape(-1), g('z_filter.running_sumsq').reshape(-1),
                                          g('z_filter.count').reshape(-1)]).to(self.device))

    # -- forward -----------------------------------------------------------------------------------
    @staticmethod
    def _flat(obs):
        if isinstance(obs, dict):
            xs = [obs['low_dim'][k] for k in obs['low_dim']]
            return xs[0] if len(xs) == 1 else torch.cat(xs, -1)
        return obs

    def _features(self, obs):
        """Pixel mode: uint8 frames [rows, C, H, W] -> CNN features (ppo_net.py:268-273,368-375)."""
        fr = obs['pixel']['camera0'] if isinstance(obs, dict) else obs
        fr = fr.reshape(-1, *fr.shape[-3:]).contiguous()
        rows = fr.shape[0]
        if getattr(self, '_stem_bufs_rows', None) != rows:
            self._stem_bufs, self._stem_bufs_rows = self.cnn_stem.buffers(rows), rows
        return self.cnn_stem.forward(fr, self._stem_bufs)

    def _no_rnn(self):
        if self.rnn_stem is not None:
            raise NotImplementedError('PPOModel.forward_actor / forward_critic run feed-forward models only; an RNN policy '
                                      'acts through PPOAgent.act and trains through PPOLearner')

    def forward_actor(self, obs, cells=None, out_pd=None):
        """-> [rows, 2A] = cat(mean, std) (builders.py:114-132), or [p | log p] of the categorical policy."""
        self._no_rnn()
        if self.cnn_stem is not None:
            mean = ops.mlp_forward(self.actor, self._features(obs))
        else:
            x = self._flat(obs)
            x2 = x.reshape(-1, x.shape[-1])
            mean = ops.mlp_forward(self.actor, x2, zf_stats=self.z_stats, zf_eps=self.z_eps)
        B, A = mean.shape[0], self.action_dim
        pd = out_pd if out_pd is not None else torch.empty(B, 2 * A, dtype=torch.float32, device=self.device)
        self.policy_pd(mean, B, pd)
        return pd

    def policy_pd(self, head_out, B, pd):
        """pd rows of the actor head's output rows: [mean | exp(log_var)], or [p | log p] of the logits."""
        if self.categorical:
            ops.cat_make_pd(head_out, B, self.action_dim, pd)
        else:
            ops.make_pd(head_out, self.log_var, B, self.action_dim, pd)

    def forward_critic(self, obs, cells=None):
        self._no_rnn()
        if self.cnn_stem is not None:
            return ops.mlp_forward(self.critic, self._features(obs))
        x = self._flat(obs)
        x2 = x.reshape(-1, x.shape[-1])
        return ops.mlp_forward(self.critic, x2, zf_stats=self.z_stats, zf_eps=self.z_eps)

    def z_update(self, obs):
        if not self.use_z_filter:
            raise ValueError('Z_update called when network is set to not use z_filter')
        x = self._flat(obs)
        x2 = x.reshape(-1, x.shape[-1])
        ops.zfilter_update(x2, x2.shape[0], self.low_dim, x2.stride(0), self.z_stats)

"""Host-side batch aggregation for experiences that arrive as Python objects (the drop-in path for
external CPU actors).  Behavioural mirror of surreal/learner/aggregator.py:33-103,106-262: same output
keys, shapes and dtypes.  Experiences produced by the on-device actors never pass through here -- the
HBM replay hands out already-batched device tensors."""
import collections

import numpy as np


def _action_type(action_spec):
    return str(action_spec['type'] if isinstance(action_spec, dict) else action_spec.type)


def _check_continuous(action_spec):
    if _action_type(action_spec) != 'continuous':
        raise NotImplementedError('action_spec unsupported ' + str(action_spec))


class SSARAggregator:
    """{obs:[s, s'], action, reward, done} list -> batched arrays (aggregator.py:52-103)."""

    def __init__(self, obs_spec, action_spec):
        assert isinstance(obs_spec, dict) and isinstance(action_spec, dict)
        _check_continuous(action_spec)
        self.obs_spec, self.action_spec = obs_spec, action_spec

    @staticmethod
    def _stack_obs(obs_list):
        out = collections.OrderedDict()
        for ob in obs_list:
            for mod in ob:
                out.setdefault(mod, collections.OrderedDict())
                for key in ob[mod]:
                    out[mod].setdefault(key, []).append(np.asarray(ob[mod][key]))
        for mod in out:
            for key in out[mod]:
                out[mod][key] = np.array(out[mod][key])
        return out

    def aggregate(self, exp_list):
        return {
            'obs': self._stack_obs([e['obs'][0] for e in exp_list]),
            'obs_next': self._stack_obs([e['obs'][1] for e in exp_list]),
            'actions': np.array([e['action'] for e in exp_list], dtype=np.float32),
            'rewards': np.expand_dims([e['reward'] for e in exp_list], axis=1),
            'dones': np.expand_dims([float(e['done']) for e in exp_list], axis=1),
        }


class MultistepAggregatorWithInfo:
    """n-step windows with per-step policy info -> batched arrays (aggregator.py:151-262).  A discrete action_spec (the
    categorical PPO policy) takes integer actions and hands the learner one-hot rows [B, n, K] float32, the layout of
    the window records."""

    def __init__(self, obs_spec, action_spec):
        assert isinstance(obs_spec, dict) and isinstance(action_spec, dict)
        t = _action_type(action_spec)
        if t not in ('continuous', 'discrete'):
            raise NotImplementedError('action_spec unsupported ' + str(action_spec))
        self.obs_spec, self.action_spec = obs_spec, action_spec
        self.n_actions = int(action_spec['dim'][0]) if t == 'discrete' else None

    def _actions(self, exp_list):
        acts = np.stack([np.stack(e['actions']) for e in exp_list])
        if self.n_actions is None:
            return acts
        K = self.n_actions
        idx = np.asarray(acts).reshape(acts.shape[0], -1)
        if idx.dtype.kind == 'f' and not np.array_equal(idx, np.round(idx)):
            raise ValueError('discrete actions must be integers')
        idx = idx.astype(np.int64)
        if idx.size and (idx.min() < 0 or idx.max() >= K):
            raise ValueError('discrete action out of range [0, %d)' % K)
        out = np.zeros(idx.shape + (K,), dtype=np.float32)
        np.put_along_axis(out, idx[..., None], 1.0, axis=-1)
        return out

    def _batch_obs(self, traj_list):
        out = {}
        for mod in self.obs_spec.keys():
            out[mod] = {}
            for key in self.obs_spec[mod].keys():
                out[mod][key] = np.stack([np.stack([ob[mod][key] for ob in traj]) for traj in traj_list])
        return out

    def aggregate(self, exp_list):
        first = exp_list[0]
        onetime = persistent = None
        if len(first['onetime_infos']) > 0:
            onetime = [np.stack([e['onetime_infos'][i] for e in exp_list]) for i in range(len(first['onetime_infos']))]
        if len(first['persistent_infos'][0]) > 0:
            persistent = [np.asarray([np.stack([step[i] for step in e['persistent_infos']]) for e in exp_list])
                          for i in range(len(first['persistent_infos'][0]))]
        return {
            'obs': self._batch_obs([e['obs'] for e in exp_list]),
            'obs_next': self._batch_obs([[e['obs_next']] for e in exp_list]),
            'actions': self._actions(exp_list),
            'rewards': np.stack([np.array(e['rewards']) for e in exp_list]),
            'persistent_infos': persistent,
            'onetime_infos': onetime,
            'dones': np.stack([np.array(e['dones']) for e in exp_list]).astype('float32'),
        }

"""Small host-side helpers shared by the plugin classes (constructor protocol, timers, trackers).

AutoInitializeMeta mirrors the reference's constructor protocol (surreal/utils/common.py:232-275):
``_initialize()`` runs after the most-derived ``__init__``.  The timers keep the names the reference
reports under (learner/base.py:160-162, replay/base.py:139-141)."""
import collections
import logging
import threading
import time
from contextlib import contextmanager


class AutoInitializeMeta(type):
    def __call__(cls, *args, **kwargs):
        obj = super().__call__(*args, **kwargs)
        if not hasattr(obj, '_initialize'):
            raise AssertionError('AutoInitializeMeta requires that subclass implements _initialize()')
        obj._initialize()
        return obj


class MovingAverageRecorder:
    """Exponential moving average with bias correction (first value seeds the average)."""

    def __init__(self, decay=0.95):
        self.decay = decay
        self.cum_value = 0.0
        self.normalization = 0.0
        self._lock = threading.Lock()

    def add_value(self, value):
        with self._lock:
            self.cum_value = self.cum_value * self.decay + value
            self.normalization = self.normalization * self.decay + 1.0
            return self.cum_value / self.normalization

    def cur_value(self):
        with self._lock:
            return self.cum_value / self.normalization if self.normalization > 0 else 0.0


class TimeRecorder:
    def __init__(self, decay=0.9995, max_seconds=10):
        self.moving_average = MovingAverageRecorder(decay)
        self.max_seconds = max_seconds
        self.started = False

    @contextmanager
    def time(self):
        t0 = time.time()
        yield None
        self.moving_average.add_value(min(self.max_seconds, time.time() - t0))

    def start(self):
        if self.started:
            raise RuntimeError('Starting a started timer')
        self.pre_time = time.time()
        self.started = True

    def lap(self):
        if not self.started:
            raise RuntimeError('Stopping a timer that is not started')
        now = time.time()
        self.moving_average.add_value(min(self.max_seconds, now - self.pre_time))
        self.pre_time = now

    def stop(self):
        self.lap()
        self.started = False

    @property
    def avg(self):
        return self.moving_average.cur_value()


class PeriodicTracker:
    """True once every ``period`` increments (surreal/session/tracker.py:10-44)."""

    def __init__(self, period, init_value=0, init_endpoint=0):
        assert isinstance(period, int) and period > 0
        self.period, self.value, self._endpoint = period, init_value, init_endpoint

    def _update(self):
        if self.value >= self._endpoint + self.period:
            self._endpoint += (self.value - self._endpoint) // self.period * self.period
            return True
        return False

    def track_increment(self, incr=1):
        self.value += incr
        return self._update()

    def track_absolute(self, value):
        self.value = value
        return self._update()


class TimedTracker:
    """True when at least ``interval`` seconds passed since the last True (utils/common.py:590-610)."""

    def __init__(self, interval):
        self.interval = interval
        self.last_time = time.time()

    def track_increment(self):
        now = time.time()
        if now - self.last_time >= self.interval:
            self.last_time = now
            return True
        return False


class ScalarSink:
    """Stand-in for the tensorplex client: keeps the last scalars per step (``add_scalars`` is the only
    call the hot path makes, learner/base.py:611; the ZMQ->TensorBoard multiplexer is out of scope)."""

    def __init__(self, name='learner'):
        self.name = name
        self.last = {}
        self.history = []
        self.keep_history = False

    def add_scalars(self, tag_to_scalar, global_step=None):
        self.last = dict(tag_to_scalar)
        if self.keep_history:
            self.history.append((global_step, dict(tag_to_scalar)))


def get_logger(name):
    log = logging.getLogger('surreal_b200.' + name)
    if not log.handlers:
        h = logging.StreamHandler()
        h.setFormatter(logging.Formatter('[%(name)s] %(message)s'))
        log.addHandler(h)
        log.setLevel(logging.WARNING)
    return log


def obs_is_pixel(obs_spec):
    """True for a pixel-only observation spec ({'pixel': {'camera0': (C, H, W)}}, docs/env.md:79-108)."""
    return 'pixel' in obs_spec and len(obs_spec['pixel']) > 0


def obs_packed_dim(obs_spec):
    """Floats per observation in the HBM staging / replay records.  Low-dim observations: the concatenated feature width.
    Pixel observations: the uint8 frame is carried as an opaque run of C*H*W/4 32-bit words (only ever COPIED by the
    windowing / replay kernels, never computed on), so frames stay uint8 in HBM: 28 224 B per 4x84x84 frame."""
    if obs_is_pixel(obs_spec):
        if 'low_dim' in obs_spec and len(obs_spec['low_dim']) > 0:
            raise NotImplementedError('mixed low_dim + pixel observations are not supported by the HBM replay records')
        shape = tuple(obs_spec['pixel']['camera0'])
        n = 1
        for v in shape:
            n *= int(v)
        if n % 16 != 0:
            raise ValueError('pixel observations need C*H*W to be a multiple of 16 bytes, got %s' % (shape,))
        return n // 4
    return sum(v[0] for v in obs_spec['low_dim'].values())


def obs_flat(obs):
    """The per-actor rows [N, packed_dim] the staging kernels copy: the low-dim feature tensor, or the uint8 frames viewed
    as 32-bit words."""
    import torch
    if isinstance(obs, dict):
        if 'low_dim' in obs and len(obs['low_dim']) > 0:
            return obs['low_dim']['flat_inputs'] if 'flat_inputs' in obs['low_dim'] else next(iter(obs['low_dim'].values()))
        fr = obs['pixel']['camera0']
        if not isinstance(fr, torch.Tensor):                      # a host env's numpy frames
            import numpy as np
            return np.ascontiguousarray(fr, dtype=np.uint8).reshape(fr.shape[0], -1).view(np.float32)
        return fr.reshape(fr.shape[0], -1).view(torch.float32)
    return obs


def obs_source(obs):
    """The array an env returned for ``obs``: the frames of a pixel observation, else obs_flat(obs) itself -- what an agent
    passes to the window wrapper's cached_device_obs."""
    if isinstance(obs, dict) and 'pixel' in obs and len(obs['pixel']) > 0 and not obs.get('low_dim'):
        return obs['pixel']['camera0']
    return obs_flat(obs)


class CellLayout(collections.namedtuple('CellLayout', 'layers hidden obs_dim')):
    """Where an RNN actor's LSTM cells sit in an observation row of the HBM staging / replay records and the learner's
    batch buffers: ``[obs (obs_dim) | h_0 .. h_{L-1} (L*H) | c_0 .. c_{L-1} (L*H)]``, i.e. the reference's
    ``onetime_infos[0 | 1]`` of shape [L, H] flattened layer-major (ppo_agent.py:133-135).  h_col / c_col: first column
    of the h / c block; width: floats per row.  At one layer this is ``[obs | h | c]``."""
    __slots__ = ()

    @property
    def h_col(self):
        return self.obs_dim

    @property
    def c_col(self):
        return self.obs_dim + self.layers * self.hidden

    @property
    def width(self):
        return self.obs_dim + 2 * self.layers * self.hidden

    def h(self, rows, k=None):
        """The h block of ``rows`` [..., width] as [..., L*H], or layer k's [..., H]."""
        o = self.h_col if k is None else self.h_col + k * self.hidden
        return rows[..., o:o + (self.layers * self.hidden if k is None else self.hidden)]

    def c(self, rows, k=None):
        o = self.c_col if k is None else self.c_col + k * self.hidden
        return rows[..., o:o + (self.layers * self.hidden if k is None else self.hidden)]


def pack_window_records(rows, obs, obs_next, frames=False, layout=None, cells=None):
    """The host packer of PPO window records ``rows`` [B, n+1, width] (DESIGN §2): ``obs`` [B, n, ...] into rows :n and
    ``obs_next`` [B, 1, ...] into row n, in the observation columns -- features, or with ``frames`` uint8 frames as their
    bytes (obs_packed_dim) -- and, for an RNN policy's CellLayout ``layout``, ``cells`` = (h, c), each [B, L, H] (the
    reference's onetime_infos: the cells of every window's first step), into the cell columns of row 0, zeros when
    ``cells`` is None.  ``rows`` is a numpy array, written in place, or a torch tensor, whose copies are issued
    non-blocking on the current stream.  Columns it does not write keep their contents."""
    import math
    import numpy as np
    import torch
    host = isinstance(rows, np.ndarray)
    as_array = np.asarray if host else torch.as_tensor

    def put(dst, src):
        src = as_array(src).reshape(dst.shape)
        if host:
            dst[...] = src
        else:
            dst.copy_(src, non_blocking=True)

    B, n, od = rows.shape[0], rows.shape[1] - 1, rows.shape[-1] if layout is None else layout.obs_dim
    obs_cols = rows.view(np.uint8 if host else torch.uint8)[..., :4 * od] if frames else rows[..., :od]
    put(obs_cols[:, :n], obs)
    put(obs_cols[:, n:], obs_next)
    if layout is None:
        return
    for i, blk in enumerate((layout.h(rows[:, 0]), layout.c(rows[:, 0]))):
        if cells is None:
            blk[...] = 0
            continue
        got = math.prod(as_array(cells[i]).shape)
        if got != B * layout.layers * layout.hidden:
            raise ValueError('onetime_infos[%d] holds %d floats; %d window(s) of a %d-layer LSTM(%d) carry [%d, %d, %d]'
                             % (i, got, B, layout.layers, layout.hidden, B, layout.layers, layout.hidden))
        put(blk, cells[i])


def rnn_cell_layout(learner_config, env_config):
    """The CellLayout of an RNN policy's records (None for a feed-forward policy): rnn_layer x rnn_hidden cells behind
    obs_packed_dim observation floats.  Raises ConfigError for rnn_layer < 1."""
    rnn = learner_config.algo.rnn if 'rnn' in learner_config.algo else None
    if rnn is None or not rnn.if_rnn_policy:
        return None
    layers = int(rnn.rnn_layer) if 'rnn_layer' in rnn else 1
    if layers < 1:
        from .session import ConfigError
        raise ConfigError('algo.rnn.rnn_layer must be at least 1, got %d' % layers)
    return CellLayout(layers, int(rnn.rnn_hidden), obs_packed_dim(env_config.obs_spec))


def record_obs_dim(learner_config, env_config):
    """Floats per observation row of the HBM staging / replay records and the learner's batch buffers: obs_packed_dim, plus
    -- for an RNN policy -- 2 * rnn_layer * rnn_hidden trailing floats that carry the actor's LSTM cells (rnn_cell_layout)
    BEFORE it acted on that observation.  The reference ships the cells of a window's first step as ``onetime_infos``
    (ppo_agent.py:133-137, exp_sender_wrapper.py:244-264); here they simply ride with every observation row."""
    lay = rnn_cell_layout(learner_config, env_config)
    return lay.width if lay is not None else obs_packed_dim(env_config.obs_spec)


def action_is_discrete(action_spec):
    """True for a discrete action spec ({'dim': (n_actions,), 'type': 'discrete'})."""
    return 'type' in action_spec and action_spec['type'] == 'discrete'


def record_action_dim(action_spec):
    """Floats per action in the HBM staging / replay records and the learner's batch buffers: the action width A of a
    continuous spec, 1 for a discrete one (the action index as a float, the [B, 1] column dqn.py:46-49 gathers with)."""
    return 1 if action_is_discrete(action_spec) else int(action_spec['dim'][0])


class LinearSchedule:
    """initial_p + min(t / schedule_timesteps, 1) (final_p - initial_p) (surreal/utils/schedule.py:76-99)."""

    def __init__(self, schedule_timesteps, final_p, initial_p=1.0):
        self.schedule_timesteps, self.final_p, self.initial_p = schedule_timesteps, final_p, initial_p

    def value(self, t):
        fraction = min(float(t) / self.schedule_timesteps, 1.0)
        return self.initial_p + fraction * (self.final_p - self.initial_p)

    def device_points(self):
        """The same schedule as PiecewiseSchedule([(0, initial_p), (T, v_T)], outside_value=v_T) with v_T = value(T)
        (initial_p + (final_p - initial_p), which may differ from final_p in the last bit): the [t_0 .. | v_0 .. |
        outside] array of sb200_dqn_act_f32, equal to value(t) at every t >= 0."""
        v_t = self.value(self.schedule_timesteps)
        return PiecewiseSchedule([(0, self.initial_p), (self.schedule_timesteps, v_t)], outside_value=v_t).device_points()


class PiecewiseSchedule:
    """Linear interpolation between (time, value) endpoints, ``outside_value`` elsewhere
    (surreal/utils/schedule.py:34-73)."""

    def __init__(self, endpoints, outside_value=None):
        idxes = [e[0] for e in endpoints]
        assert idxes == sorted(idxes)
        self._endpoints, self._outside_value = list(endpoints), outside_value

    def value(self, t):
        for (l_t, l), (r_t, r) in zip(self._endpoints[:-1], self._endpoints[1:]):
            if l_t <= t < r_t:
                alpha = float(t - l_t) / (r_t - l_t)
                return l + alpha * (r - l)
        assert self._outside_value is not None
        return self._outside_value

    def device_points(self):
        ts = [float(e[0]) for e in self._endpoints]
        vs = [float(e[1]) for e in self._endpoints]
        return ts + vs + [float(self._outside_value)]

"""Host staging (surreal_b200.staging) and the one host encoding of PPO window records (utils.pack_window_records):

  * the pool's pinned rule for every staged dtype: a pinned, C-contiguous, writeable array of the dtype is used by its own
    address, anything else is copied into the named pinned buffer, which later calls reuse; upload() counts PCIe bytes;
  * the same windows given to PPOLearner.learn as a numpy batch, as a CPU-tensor batch and through FIFOReplay.insert +
    sample give the learner bit-identical batch buffers (MLP, pixel and 2-layer RNN policies); likewise numpy batches and
    UniformReplay.insert + sample for the off-policy learner."""
import random

import numpy as np
import pytest
import torch

from helpers import ddpg_configs, ppo_configs

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64, np.uint8, np.int64]


def _pinned_array(values, dtype):
    a = torch.empty(values.shape, dtype=torch.from_numpy(np.empty(0, dtype)).dtype, pin_memory=True).numpy()
    a[...] = values
    return a


@pytest.mark.parametrize('dtype', DTYPES, ids=lambda d: np.dtype(d).name)
def test_pool_passes_pinned_arrays_and_stages_the_rest(dtype):
    from surreal_b200.staging import Staging
    st = Staging(torch.device('cuda', 0))
    shape = (4, 6)
    vals = np.random.default_rng(0).integers(0, 100, size=shape)       # exact in every staged dtype
    own = _pinned_array(vals, dtype)
    assert st.host_ptr('x', own, shape, dtype).value == own.ctypes.data
    wide = _pinned_array(np.repeat(vals, 2, axis=1), dtype)
    read_only = _pinned_array(vals, dtype)
    read_only.flags.writeable = False
    other = np.float32 if np.dtype(dtype) == np.float64 else np.float64
    staged = {'unpinned': vals.astype(dtype), 'wrong dtype': _pinned_array(vals, other),
              'non-contiguous': wide[:, ::2], 'read-only': read_only}
    addrs = set()
    for why, arr in staged.items():
        p = st.host_ptr('x', arr, shape, dtype).value
        pin = st.pinned('x', shape, dtype)
        assert p == pin.data_ptr() and p != arr.ctypes.data, why
        assert np.array_equal(pin.numpy(), np.asarray(arr, dtype).reshape(shape)), why
        addrs.add(p)
    assert len(addrs) == 1                                              # one buffer, reused by every call
    dev = st.device('x', shape, dtype)
    assert st.device('x', shape, dtype) is dev
    assert st.upload('x', torch.from_numpy(vals.astype(dtype)), dev) == dev.numel() * dev.element_size()
    src = torch.from_numpy(vals.astype(dtype)).cuda() + 1
    assert st.upload('x', src, dev) == 0
    assert st.upload('x', dev, dev) == 0
    torch.cuda.synchronize()
    assert torch.equal(dev, src)
    for arr in (own, staged['unpinned']):
        assert st.upload('x', arr, dev) == dev.numel() * dev.element_size()
        torch.cuda.synchronize()
        assert np.array_equal(dev.cpu().numpy(), vals.astype(dtype))


def _ppo_cfg(kind, n, B, A):
    lc, ec, sc = ppo_configs(D=6, A=A, n_step=n, stride=n, B=B, memory_size=4 * B, use_z=False)
    if kind == 'pixel':
        ec.obs_spec = {'pixel': {'camera0': (2, 20, 20)}}
        ec.pixel_input = True
        lc.model.cnn_feature_dim = 16
    if kind == 'rnn2':
        lc.algo.rnn.if_rnn_policy = True
        lc.algo.rnn.horizon, lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = 2, 5, 2
    return lc, ec, sc


@pytest.mark.parametrize('kind', ['mlp', 'pixel', 'rnn2'])
def test_ppo_host_batches_and_fifo_inserts_ingest_the_same_records(kind):
    from surreal_b200.learner import PPOLearner
    from surreal_b200.replay import FIFOReplay
    n, B, A, L_, H = 4, 5, 2, 2, 5
    lc, ec, sc = _ppo_cfg(kind, n, B, A)
    rng = np.random.default_rng(1)
    if kind == 'pixel':
        obs = rng.integers(0, 256, size=(B, n + 1, 2, 20, 20), dtype=np.uint8)
        key = lambda x: {'pixel': {'camera0': x}}                           # noqa: E731
    else:
        obs = rng.standard_normal((B, n + 1, 6)).astype(np.float32)
        key = lambda x: {'low_dim': {'flat_inputs': x}}                     # noqa: E731
    act = rng.standard_normal((B, n, A)).astype(np.float32)
    pd = rng.standard_normal((B, n, 2 * A)).astype(np.float32)
    rew = rng.standard_normal((B, n))                                       # float64, rounded once on ingest
    done = rng.random((B, n)) < 0.3
    cells = [rng.standard_normal((B, L_, H)).astype(np.float32) for _ in range(2)] if kind == 'rnn2' else None
    batch = {'obs': key(obs[:, :n]), 'obs_next': key(obs[:, n:]), 'actions': act, 'rewards': rew, 'dones': done,
             'persistent_infos': [pd], 'onetime_infos': cells}
    tensors = {'obs': key(torch.from_numpy(obs[:, :n])), 'obs_next': key(torch.from_numpy(obs[:, n:])),
               'actions': torch.from_numpy(act), 'rewards': torch.from_numpy(rew), 'dones': torch.from_numpy(done),
               'persistent_infos': [torch.from_numpy(pd)],
               'onetime_infos': None if cells is None else [torch.from_numpy(c) for c in cells]}
    R = FIFOReplay(lc, ec, sc)
    for b in range(B):
        R.insert({'obs': [key(obs[b, t]) for t in range(n)], 'obs_next': key(obs[b, n]),
                  'actions': list(act[b]), 'rewards': list(rew[b]), 'dones': list(done[b]),
                  'persistent_infos': [[pd[b, t]] for t in range(n)],
                  'onetime_infos': None if cells is None else [cells[0][b], cells[1][b]]})
    got = []
    for src in (batch, tensors, R.sample(B)):
        learner = PPOLearner(lc, ec, sc)
        learner._preprocess_batch_ppo(src)
        torch.cuda.synchronize()
        got.append([t.cpu() for t in (learner._obs_full, learner._actions, learner._pds, learner._rewards, learner._dones)])
    for other in got[1:]:
        for a, b in zip(got[0], other):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    rows = got[0][0]
    if kind == 'pixel':
        assert np.array_equal(rows.view(torch.uint8).numpy().reshape(obs.shape), obs)
    else:
        assert np.array_equal(rows[:, :, :6].numpy(), obs)
    if cells is not None:
        cl = learner.cell_layout
        assert np.array_equal(cl.h(rows[:, 0]).numpy().reshape(B, L_, H), cells[0])
        assert np.array_equal(cl.c(rows[:, 0]).numpy().reshape(B, L_, H), cells[1])
    assert np.array_equal(got[0][3].numpy(), rew.astype(np.float32))


def test_off_policy_host_batches_and_uniform_inserts_ingest_the_same_rows():
    from surreal_b200.learner import DDPGLearner
    from surreal_b200.replay import UniformReplay
    D, A, B = 9, 3, 16
    lc, ec, sc = ddpg_configs(D=D, A=A, B=B, memory_size=64)
    rng = np.random.default_rng(2)
    s, s1 = rng.standard_normal((B, D)), rng.standard_normal((B, D)).astype(np.float32)
    a, r, d = rng.standard_normal((B, A)).astype(np.float32), rng.standard_normal(B), rng.random(B) < 0.3
    R = UniformReplay(lc, ec, sc)
    for i in range(B):
        R.insert({'obs': [{'low_dim': {'flat_inputs': s[i]}}, {'low_dim': {'flat_inputs': s1[i]}}], 'action': a[i],
                  'reward': r[i], 'done': d[i]})
    random.seed(3)
    sampled = R.sample(B)
    idx = sampled['indices'].numpy()
    host = {'obs': s[idx], 'obs_next': s1[idx], 'actions': a[idx], 'rewards': r[idx].reshape(B, 1),
            'dones': d[idx].reshape(B, 1)}
    got = []
    for src in (host, sampled):
        learner = DDPGLearner(lc, ec, sc)
        learner.preprocess(src)
        torch.cuda.synchronize()
        got.append({k: v.cpu() for k, v in learner._own.items()})
    for k in got[0]:
        assert torch.equal(got[0][k].view(torch.int32), got[1][k].view(torch.int32)), k
    assert np.array_equal(got[0]['obs'].numpy(), s[idx].astype(np.float32))

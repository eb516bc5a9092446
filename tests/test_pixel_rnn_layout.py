"""Host-side layout of CNN + LSTM records (no GPU): a pixel RNN policy's record row is [frame words | h | c], and a host
env's numpy frames become those words bit for bit."""
import numpy as np
import torch

from helpers import ppo_configs


def _cfg(C=4, HW=84, H=100, layers=1):
    lc, ec, sc = ppo_configs(D=1, use_z=False)
    ec.obs_spec = {'pixel': {'camera0': (C, HW, HW)}}
    ec.pixel_input = True
    lc.algo.rnn.if_rnn_policy = True
    lc.algo.rnn.rnn_hidden, lc.algo.rnn.rnn_layer = H, layers
    return lc, ec


def test_pixel_rnn_record_width_and_cell_columns():
    from surreal_b200.utils import record_obs_dim, rnn_cell_layout
    lc, ec = _cfg(layers=2)
    cl = rnn_cell_layout(lc, ec)
    assert cl.obs_dim == 4 * 84 * 84 // 4 == 7056
    assert record_obs_dim(lc, ec) == 7056 + 2 * 2 * 100 == cl.width
    row = np.arange(cl.width, dtype=np.float32)
    assert cl.h(row, 1)[0] == 7056 + 100 and cl.c(row, 0)[0] == 7056 + 200


def test_host_frames_become_their_words_bit_for_bit():
    from surreal_b200.utils import obs_flat, obs_source
    fr = np.random.default_rng(0).integers(0, 256, size=(3, 2, 20, 20), dtype=np.uint8)
    fr[0, 0, 0, :4] = [0x01, 0x00, 0xc0, 0x7f]            # a quiet-NaN word with a payload
    obs = {'pixel': {'camera0': fr}}
    w = obs_flat(obs)
    assert w.dtype == np.float32 and w.shape == (3, 200)
    assert np.array_equal(w.view(np.uint8).reshape(fr.shape), fr)
    assert obs_source(obs) is fr
    dev_like = {'pixel': {'camera0': torch.from_numpy(fr)}}
    assert torch.equal(obs_flat(dev_like).view(torch.uint8).reshape(fr.shape), torch.from_numpy(fr))
    low = {'low_dim': {'flat_inputs': np.zeros((3, 5), np.float32)}}
    assert obs_source(low) is low['low_dim']['flat_inputs']

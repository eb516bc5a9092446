"""The device sampler of UniformReplay (sb200_uniform_sample_gather_f32 / sb200_uniform_view), restated on the CPU.

``device_sample_indices`` is the oracle of the kernel's index stream, on top of oracle/philox.py: Philox call p keyed
(seed, draw counter, p) serves draws 2p (words x:y) and 2p+1 (words z:w); a draw is floor(u * count / 2^64) of its 64
bits, mapped to ring slot (start + r) % capacity.  ``sampling_view`` is the rule of sb200_uniform_view.  The GPU tests
(test_ddpg_device_engine_gpu.py) compare the kernels with both, bit for bit; here the restatement itself is checked."""
import numpy as np
import pytest

from oracle.philox import philox4x32_10

COUNTS = [1, 2, 5, 96, 3000, 2 ** 20, 2 ** 20 + 1]


def device_draws(seed, counter, count, batch):
    """-> list of ``batch`` Python ints in [0, count): the draws before the ring mapping."""
    calls = np.arange((batch + 1) // 2, dtype=np.uint64)
    x, y, z, w = philox4x32_10(np.uint64(seed), np.uint64(counter), calls)
    out = []
    for i in range(batch):
        hi, lo = (x, y) if i % 2 == 0 else (z, w)
        u = (int(hi[i // 2]) << 32) | int(lo[i // 2])
        out.append((u * int(count)) >> 64)
    return out


def device_sample_indices(seed, counter, start, count, capacity, batch):
    """-> int64 array [batch]: the ring slots one sampler launch draws at draw counter ``counter``."""
    return np.array([(int(start) + r) % int(capacity) for r in device_draws(seed, counter, count, batch)], dtype=np.int64)


def sampling_view(next_idx, size, capacity, reserve):
    """-> (start, count): the filled slots that the next ``reserve`` inserts cannot overwrite."""
    if size + reserve <= capacity:
        return 0, size
    return (next_idx + reserve) % capacity, capacity - reserve


def test_philox_known_answer():
    """Random123's published known-answer vectors for philox4x32_10."""
    assert [int(v) for v in philox4x32_10(0, 0, 0)] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    ones = np.uint64(0xFFFFFFFFFFFFFFFF)
    assert [int(v) for v in philox4x32_10(ones, ones, ones)] == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]


def test_two_draws_by_hand():
    """seed 0, counter 0, call 0 is the all-zero known answer: u0 = 0x6627e8d5e169c58d = 0.39904...* 2^64 and
    u1 = 0xbc57ac4c9b00dbd8 = 0.73571... * 2^64.  Over 96 records: floor(38.3) = 38 and floor(70.6) = 70; in a view that
    starts at slot 90 of a 100-slot ring they are slots 28 and 60."""
    assert device_draws(0, 0, 96, 2) == [38, 70]
    assert device_sample_indices(0, 0, 90, 96, 100, 2).tolist() == [28, 60]
    assert device_sample_indices(0, 0, 0, 96, 100, 1).tolist() == [38]            # an odd batch uses half a call


@pytest.mark.parametrize('count', COUNTS)
def test_draws_stay_in_range_and_reach_both_ends(count):
    d = np.array(device_draws(11, 3, count, 4096))
    assert d.min() >= 0 and d.max() < count
    if count <= 96:
        assert set(d.tolist()) == set(range(count))
    s = device_sample_indices(11, 3, count // 2, count, count + 7, 4096)
    assert s.min() >= 0 and s.max() < count + 7
    assert np.array_equal(s, (count // 2 + d) % (count + 7))


def test_counter_and_seed_select_different_streams():
    a = device_draws(5, 0, 3000, 64)
    assert a != device_draws(5, 1, 3000, 64) and a != device_draws(6, 0, 3000, 64)
    assert a == device_draws(5, 0, 3000, 64)
    assert a[:10] == device_draws(5, 0, 3000, 10)          # draw i does not depend on the batch size


def test_chi_square_of_a_million_draws():
    from scipy.stats import chi2
    n, bins, count = 2 ** 20, 64, 3000 * 64
    d = np.array(device_draws(2024, 7, count, n), dtype=np.int64)
    hist = np.bincount(d * bins // count, minlength=bins)
    stat = float(((hist - n / bins) ** 2 / (n / bins)).sum())
    assert chi2.ppf(1e-4, bins - 1) < stat < chi2.ppf(1 - 1e-4, bins - 1), stat


@pytest.mark.parametrize('capacity,reserve', [(10, 3), (10, 5), (16, 1), (12, 0)])
def test_view_rule_against_a_ring_being_written(capacity, reserve):
    """Brute force: a ring whose slot k % capacity holds insert k.  For every fill level up to three times around, the
    view holds only filled slots, none of them changes while up to ``reserve`` more records arrive, and no other
    filled slot survives all ``reserve`` of them (the view is as large as it can be)."""
    for total in range(0, 3 * capacity + 1):
        ring = {k % capacity: k for k in range(total)}
        next_idx, size = total % capacity, min(total, capacity)
        start, count = sampling_view(next_idx, size, capacity, reserve)
        view = [(start + r) % capacity for r in range(count)]
        assert len(set(view)) == count and all(s in ring for s in view)
        after = dict(ring)
        for k in range(total, total + reserve):
            after[k % capacity] = k
            assert all(after[s] == ring[s] for s in view), (total, k)
        assert count == sum(1 for s in ring if after[s] == ring[s])

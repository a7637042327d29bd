"""-m gpu: the seed sort on 64-bit words (keys of <= 64 bits) against a stable numpy sort and against
the 128-bit passes, through fgb_seeds_from_records on device buffers."""
import numpy as np
import pytest

from fastga_b200 import lib

pytestmark = pytest.mark.gpu

#  field widths (anti, band, jcont, icont) for a key of 12 + sum + 1 bits; 22: two passes, the narrow plan
#  with no middle pass (16 -> 8 bytes, then 8 -> 16)
BITS = {14: (1, 0, 0, 0), 22: (9, 0, 0, 0), 57: (22, 16, 3, 3), 63: (25, 19, 3, 3), 64: (25, 19, 3, 4),
        80: (30, 24, 6, 7)}
#  tile sizes of the narrowing pass (4096) and of the passes on 8-byte words (8192)
SIZES = (0, 1, 2, 4095, 4096, 4097, 8191, 8192, 8193, 2 * 8192 + 3, 3_000_017)


def random_records(rng, n, key):
    recs = np.zeros((n, 2), dtype=np.uint64)
    recs[:, 0] = rng.integers(0, 1 << 64, size=n, dtype=np.uint64, endpoint=False)
    if key < 64:
        recs[:, 0] &= np.uint64((1 << key) - 1)
    if key > 64:
        recs[:, 1] = rng.integers(0, 1 << (key - 64), size=n, dtype=np.uint64)
    return recs


def stable_sorted(recs):
    """stable order on bits [6, key): the lcp field (bits 0..5) never takes part"""
    return recs[np.lexsort((recs[:, 0] >> np.uint64(6), recs[:, 1]))]


def sort_on_device(recs, key):
    import torch
    d = torch.from_numpy(recs.view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    s = lib.seeds_from_records(d.data_ptr() if len(recs) else 0, len(recs), BITS[key], 1, 1)
    out = s.download()
    assert s.n == len(recs)
    return out


@pytest.mark.parametrize("key", [14, 22, 57, 63, 64])
def test_seed_sort_matches_stable_numpy_sort(key):
    rng = np.random.default_rng(key)
    for n in SIZES:
        recs = random_records(rng, n, key)
        assert np.array_equal(sort_on_device(recs, key), stable_sorted(recs)), (key, n)


@pytest.mark.parametrize("key", [57, 63, 64])
def test_seed_sort_keeps_input_order_of_equal_keys(key):
    """few distinct keys, each many times with random lcp bits across many tiles: only a stable sort
    returns them in input order"""
    rng = np.random.default_rng(100 + key)
    for n in (8193, 300_001):
        keys = random_records(rng, 7, key)[:, 0] & ~np.uint64(63)
        recs = np.zeros((n, 2), dtype=np.uint64)
        recs[:, 0] = keys[rng.integers(0, len(keys), size=n)] | rng.integers(0, 64, size=n, dtype=np.uint64)
        assert np.array_equal(sort_on_device(recs, key), stable_sorted(recs)), (key, n)


def test_key_above_64_bits_sorts_with_the_hi_word():
    rng = np.random.default_rng(80)
    for n in (4097, 500_003):
        recs = random_records(rng, n, 80)
        assert recs[:, 1].any()
        assert np.array_equal(sort_on_device(recs, 80), stable_sorted(recs)), n


def test_records_with_hi_bits_under_a_64_bit_key_are_refused():
    """the 64-bit passes drop the hi word: records that carry one anyway must fail the call, never come
    back mis-ordered"""
    rng = np.random.default_rng(9)
    recs = random_records(rng, 20_000, 63)
    recs[12_345, 1] = 1
    with pytest.raises(lib.FgbError):
        sort_on_device(recs, 63)


def test_64_bit_and_128_bit_passes_give_identical_handles(small_pair, monkeypatch):
    gA, gB = small_pair
    dA, dB = lib.DeviceGenome(gA), lib.DeviceGenome(gB)
    xA, xB = lib.DeviceGix.build(dA), lib.DeviceGix.build(dB)
    amx, bmx = int(gA.clen.max()), int(gB.clen.max())
    ptr, n, bits, sumlen, _ = lib.seeds_merge(xA, xB, amx, bmx, 10)
    try:
        assert 12 + sum(bits) + 1 <= 64 and n > 2 * 8192
        narrow = lib.seeds_from_records(ptr, n, bits, amx, bmx, sumlen)
        monkeypatch.setenv("FGB_SEED_SORT_WIDE", "1")
        wide = lib.seeds_from_records(ptr, n, bits, amx, bmx, sumlen)
        monkeypatch.delenv("FGB_SEED_SORT_WIDE")
    finally:
        lib.device_free(ptr)
    got, want = narrow.download(), wide.download()
    assert got.shape == (n, 2) and not got[:, 1].any()
    assert got.tobytes() == want.tobytes()
    assert got.tobytes() == lib.DeviceSeeds.find(xA, xB, amx, bmx, 10).download().tobytes()

"""-m gpu: the pair adaptamer merge (merge.cu adaptamer_merge_kernel) on the crafted table pairs of
pair_cases.py, record by record against the oracle's merge (itself pinned to the reference on the same
tables, test_pair_cases.py).  Per case and f:
  * both tables uploaded (the device builds the prefix index and the LCP bytes), the index equal to the case's;
  * lib.DeviceSeeds.find under both seed-sort plans: count, sum of seed lengths and the sorted records;
  * lib.seeds_merge, the unsorted route of the sharded path: count, sum, the forward T1 entries merged, and
    its records sorted by fgb_seeds_from_records (from bit 6).
What each case reaches in the kernel (tile, staging, write-out, byte loop, rounds) is in pair_cases.py."""
import os

import numpy as np
import pytest

import oracle_lib as ol
import pair_cases as pc
from fastga_b200 import lib

pytestmark = pytest.mark.gpu

LOW6 = np.array([~np.uint64(63), ~np.uint64(0)], dtype=np.uint64)     # the lcp field does not order seeds


def _find(x1, x2, c, freq, wide):
    old = os.environ.get("FGB_SEED_SORT_WIDE")
    os.environ["FGB_SEED_SORT_WIDE"] = "1" if wide else "0"
    try:
        return lib.DeviceSeeds.find(x1, x2, c.amx, c.bmx, freq)
    finally:
        if old is None:
            del os.environ["FGB_SEED_SORT_WIDE"]
        else:
            os.environ["FGB_SEED_SORT_WIDE"] = old


def _same_records(got, want, what):
    # sorted on everything above the lcp field; seeds equal there are the same pair of posts
    assert np.array_equal(got & LOW6, want & LOW6), what
    o = np.lexsort((got[:, 0], got[:, 1]))
    assert np.array_equal(got[o], want), what


def _upload(T, c, which):
    pb, cb = c.upload_bytes(which)
    return lib.DeviceGix.upload(T, pb, cb, len(c.clen1 if which == 1 else c.clen2))


@pytest.mark.parametrize("name", sorted(pc.CASES))
def test_pair_merge_on_crafted_tables(name):
    c = pc.case(name)
    pstart2 = c.pstart2()
    x1, x2 = _upload(c.T1, c, 1), _upload(c.T2, c, 2)
    try:
        for x, T, ps in ((x1, c.T1, pc.pstart_of(c.T1)), (x2, c.T2, pstart2)):
            tab, pstart, _ = x.download()
            assert np.array_equal(tab, T) and np.array_equal(pstart, ps)
        for freq in c.freqs:
            seeds, sumlen = ol.merge(c.T1, c.T2, pstart2, freq)
            if name in ("overflow", "packed_ceiling"):
                # more seeds than the first reservation: the merge ran a second time
                assert len(seeds) > pc.first_reservation(c.n1)
            want = None
            for wide in (False, True):
                ds = _find(x1, x2, c, freq, wide)
                try:
                    assert (ds.n, ds.sumlen) == (len(seeds), sumlen), (freq, wide)
                    if want is None:
                        want = ol.seed_records(seeds, ds.layout + (c.amx, c.bmx), sort=True)
                    _same_records(ds.download(), want, (freq, wide))
                finally:
                    ds.close()
            # the sharded path's route: unsorted records, then its own sort from bit 6
            ptr, n, bits, sl, n1m = lib.seeds_merge(x1, x2, c.amx, c.bmx, freq)
            try:
                assert (n, sl, n1m) == (len(seeds), sumlen, c.n1), freq
                ds = lib.seeds_from_records(ptr, n, bits, c.amx, c.bmx, sl)
                try:
                    assert ds.n == n
                    _same_records(ds.download(), want, (freq, "seeds_merge"))
                finally:
                    ds.close()
            finally:
                if ptr:
                    lib.device_free(ptr)
    finally:
        x1.close()
        x2.close()

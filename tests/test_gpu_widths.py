"""-m gpu: the stages against the oracle on the width cases of tests/edge_cases.py, where packed fields
change size: seed keys past 64 bits (fields in the upper word, the 128-bit sort passes), contig ranks
wider than 8 bits, positions past 2^24, 32767 contigs.  Also the genome limits of fgb_genome_create."""
import ctypes as C
import os

import numpy as np
import pytest

import edge_cases
import oracle_lib as ol
from fastga_b200 import formats, lib, load_library

pytestmark = pytest.mark.gpu
WIDE = ["seed_key_65", "icont_straddles", "long_and_many", "max_contigs"]


@pytest.fixture(scope="module")
def staged():
    """case name -> (genomes, device genomes, device tables), built once per module, one case at a time"""
    cache = {}

    def get(name):
        if name not in cache:
            cache.clear()
            A, B, _, _ = edge_cases.CASES[name]()
            gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
            dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
            cache[name] = (gA, gB, dA, dB, lib.DeviceGix.build(dA), lib.DeviceGix.build(dB))
        return cache[name]
    yield get
    cache.clear()


def _seeds(gA, gB, xA, xB):
    amx, bmx = int(gA.clen.max()), int(gB.clen.max())
    return lib.DeviceSeeds.find(xA, xB, amx, bmx, 10)


@pytest.mark.parametrize("name", WIDE)
def test_tables_match_oracle_at_wide_fields(name, staged):
    """k-mer tables with 2-byte contig fields, 4-byte posts, 32767 ranks (length ties among the
    max_contigs fillers: ranks come from the device's own sort, which must still be by length)"""
    gA, gB, dA, dB, xA, xB = staged(name)
    for g, dg, x, want_bytes in ((gA, dA, xA, edge_cases.REGIMES[name]["gixA"]),
                                 (gB, dB, xB, edge_cases.REGIMES[name]["gixB"])):
        assert (np.diff(g.clen[dg.perm]) <= 0).all()
        assert (x.post_bytes, x.cont_bytes) == formats.gix_bytes(g) == want_bytes
        want, wstart = ol.gix_build(g, dg.crank)
        tab, pstart, _ = x.download()
        assert x.n == len(want)
        assert np.array_equal(tab, want)
        assert np.array_equal(pstart, wstart)


@pytest.mark.parametrize("name", WIDE)
def test_seeds_match_oracle_at_wide_keys(name, staged):
    gA, gB, dA, dB, xA, xB = staged(name)
    ds = _seeds(gA, gB, xA, xB)
    tA, _, _ = xA.download(False)
    tB, pB, _ = xB.download()
    seeds, sumlen = ol.merge(tA, tB, pB, 10)
    assert ds.n == len(seeds) > 1000 and ds.sumlen == sumlen
    layout = ol.seed_layout(gA, gB)
    assert ds.layout == layout[:4] and 13 + sum(layout[:4]) == edge_cases.REGIMES[name]["key"]
    got = ds.download()
    assert np.array_equal(got, ol.seed_records(seeds, layout, sort=True))
    assert (got[:, 1] != 0).any() == (13 + sum(layout[:4]) > 64)


@pytest.mark.parametrize("name", WIDE)
def test_extend_matches_oracle_at_wide_keys(name, staged):
    """the chain scan + extension reads contig ranks, diagonals and strand out of records whose upper
    fields straddle bit 64: same records as the oracle, in the same discovery order"""
    from test_gpu_stages import _canon
    gA, gB, dA, dB, xA, xB = staged(name)
    ds = _seeds(gA, gB, xA, xB)
    seeds = ds.download()
    layout = ds.layout + (int(gA.clen.max()), int(gB.clen.max()))
    want, wpool, whits = ol.search(seeds, layout, gA, gB, dA.perm, dB.perm, gA.freq)
    ov = lib.DeviceOverlaps.extend(ds, dA, dB, gA.freq)
    got, gpool = ov.records()
    assert ov.counters()["hits"] == whits
    jb, ib = layout[2], layout[3]
    pk = got["pairkey"].astype(np.int64)
    jc = pk & ((1 << jb) - 1)
    ic = (pk >> jb) & ((1 << ib) - 1)
    comp = pk >> (jb + ib)
    g = _canon(got, gpool, dA.perm[ic], dB.perm[jc], comp)
    w = _canon(want, wpool)
    assert len(w) > 20 and g == w


def test_narrow_and_wide_seed_sorts_give_identical_handles_at_64_bit_keys(staged):
    """a 64-bit key is the widest the 64-bit passes take: same handle as the 128-bit passes, and the
    oracle's records"""
    gA, gB, dA, dB, xA, xB = staged("seed_key_64")
    narrow = _seeds(gA, gB, xA, xB)
    assert 13 + sum(narrow.layout) == 64
    os.environ["FGB_SEED_SORT_WIDE"] = "1"
    try:
        wide = _seeds(gA, gB, xA, xB)
    finally:
        del os.environ["FGB_SEED_SORT_WIDE"]
    a, b = narrow.download(), wide.download()
    assert a.tobytes() == b.tobytes() and not a[:, 1].any()
    tA, _, _ = xA.download(False)
    tB, pB, _ = xB.download()
    seeds, _ = ol.merge(tA, tB, pB, 10)
    assert np.array_equal(a, ol.seed_records(seeds, ol.seed_layout(gA, gB), sort=True))


def _genome_create(nc, clen, bps):
    L = load_library()
    clen = np.ascontiguousarray(clen, dtype=np.int64)
    boff = np.zeros(len(clen), dtype=np.int64)
    h = C.c_void_p()
    rc = L.fgb_genome_create(bps.ctypes.data, bps.size, nc, clen.ctypes.data, boff.ctypes.data, 0, C.byref(h), None)
    return rc, h


def test_genome_limits_are_refused_before_anything_is_allocated():
    """contig ranks are 15-bit fields: 32767 contigs are accepted, 32768 refused; a contig length of
    2^31 - 1 is refused before its bases are read (the buffer passed here holds 16 bytes)"""
    live = lib.device_live_bytes()
    rc, h = _genome_create(0x8000, np.full(0x8000, 4), np.zeros(0x8000, np.uint8))
    assert rc == -3 and not h.value
    assert lib.device_live_bytes() == live
    rc, h = _genome_create(1, [(1 << 31) - 1], np.zeros(16, np.uint8))
    assert rc == -3 and not h.value
    assert lib.device_live_bytes() == live
    g = formats.genome_from_arrays([np.full(4 + (k & 7), k & 3, np.uint8) for k in range(0x7fff)])
    dg = lib.DeviceGenome(g)
    assert len(dg.perm) == 0x7fff and (np.diff(g.clen[dg.perm]) <= 0).all()
    dg.close()
    assert lib.device_live_bytes() == live

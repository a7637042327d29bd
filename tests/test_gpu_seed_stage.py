"""-m gpu: the seed stage between the merge and the extension launch.  Records that a merge built are
sorted from bit 7 (bit 6, the low bit of the diagonal, is bit 12 XOR a constant of the strand), records
from a caller from bit 6; the band segments, the work list and the chunk plan are built on the device.
Checked against the oracle's merge and chain scan and against a numpy restatement of the segments and
the work order."""
import os

import numpy as np
import pytest

import oracle_lib as ol
from fastga_b200 import formats, lib, synth

pytestmark = pytest.mark.gpu

PREF_LONG = 64                  # a work triple with more seeds is scanned in chunks
CHUNK = 1536                    # merged seeds per chunk of fgb_extend
HCAP = 48                       # hits a chunk records


def _revcomp(a):
    return (3 - a[::-1]).astype(np.uint8)


def _parity_pair(amx_odd, bmx_odd, seed):
    """two contigs each side, the second of B reverse-complemented (seeds on both strands); the longest
    contig of A has amx_odd parity, of B bmx_odd"""
    rng = np.random.default_rng(seed)
    A = [rng.integers(0, 4, 260_000 + amx_odd, dtype=np.uint8), rng.integers(0, 4, 150_001, dtype=np.uint8)]
    B = [synth.diverged_copy(rng, A[0], 0.04, sv_every=50_000, inversions=False),
         _revcomp(synth.diverged_copy(rng, A[1], 0.04, sv_every=50_000, inversions=False))]
    if len(B[0]) % 2 != bmx_odd:
        B[0] = B[0][:-1]
    assert len(B[0]) > len(B[1])
    return A, B


def _wide(on):
    if on:
        os.environ["FGB_SEED_SORT_WIDE"] = "1"
    else:
        os.environ.pop("FGB_SEED_SORT_WIDE", None)


def _strand(recs, layout):
    """the key's top bit, and a check that bit 6 XOR bit 12 is one value per strand"""
    key = 12 + sum(layout[:4]) + 1
    lo, hi = recs[:, 0], recs[:, 1]
    top = key - 1
    strand = ((lo >> np.uint64(top)) if top < 64 else (hi >> np.uint64(top - 64))) & np.uint64(1)
    par = ((lo >> np.uint64(6)) ^ (lo >> np.uint64(12))) & np.uint64(1)
    for s in (0, 1):
        assert len(np.unique(par[strand == s])) <= 1, s
    return strand


@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("amx_odd,bmx_odd", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_pair_seeds_from_bit7_match_oracle_and_bit6_sort(amx_odd, bmx_odd, wide):
    A, B = _parity_pair(amx_odd, bmx_odd, 40 + 2 * amx_odd + bmx_odd)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    amx, bmx = int(gA.clen.max()), int(gB.clen.max())
    assert (amx % 2, bmx % 2) == (amx_odd, bmx_odd)
    dA, dB = lib.DeviceGenome(gA), lib.DeviceGenome(gB)
    xA, xB = lib.DeviceGix.build(dA), lib.DeviceGix.build(dB)
    try:
        _wide(wide)
        ds = lib.DeviceSeeds.find(xA, xB, amx, bmx, 10)
        got = ds.download()
        tA, _, _ = xA.download(False)
        tB, pB, _ = xB.download()
        seeds, sumlen = ol.merge(tA, tB, pB, 10)
        assert ds.n == len(seeds) and ds.sumlen == sumlen
        assert np.array_equal(got, ol.seed_records(seeds, ds.layout + (amx, bmx), sort=True))
        strand = _strand(got, ds.layout)
        assert (strand == 0).any() and (strand == 1).any()
        # the same merged records sorted from bit 6 through fgb_seeds_from_records
        ptr, n, bits, sl, _ = lib.seeds_merge(xA, xB, amx, bmx, 10)
        try:
            s6 = lib.seeds_from_records(ptr, n, bits, amx, bmx, sl)
            assert np.array_equal(s6.download(), got)
            s6.close()
        finally:
            lib.device_free(ptr)
        ds.close()
    finally:
        _wide(False)
        for h in (xA, xB, dA, dB):
            h.close()


@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("amx_odd", [0, 1])
def test_self_seeds_from_bit7_match_oracle(amx_odd, wide):
    rng = np.random.default_rng(60 + amx_odd)
    a = rng.integers(0, 4, 200_000 + amx_odd, dtype=np.uint8)
    A = [a, synth.diverged_copy(rng, a[:120_000], 0.03, sv_every=40_000, inversions=False),
         _revcomp(synth.diverged_copy(rng, a[50_000:140_001], 0.03, sv_every=40_000, inversions=False))]
    g = formats.genome_from_arrays(A)
    amx = int(g.clen.max())
    assert amx % 2 == amx_odd
    d = lib.DeviceGenome(g, want_revcomp=True)
    x = lib.DeviceGix.build(d)
    try:
        _wide(wide)
        ds = lib.DeviceSeeds.find_self(x, amx, 10)
        got = ds.download()
        tab, pstart, _ = x.download()
        seeds, sumlen = ol.self_merge(tab, pstart, 10)
        assert (ds.n, ds.sumlen) == (len(seeds), sumlen)
        want = ol.seed_records(seeds, ds.layout + (amx, amx), sort=True)
        # sorted on everything above the lcp field; seeds equal there are the same pair of posts
        low6 = np.array([~np.uint64(63), ~np.uint64(0)], dtype=np.uint64)
        assert np.array_equal(got & low6, want & low6)
        assert np.array_equal(got[np.lexsort((got[:, 0], got[:, 1]))], want)
        strand = _strand(got, ds.layout)
        assert (strand == 0).any() and (strand == 1).any()
        ds.close()
    finally:
        _wide(False)
        x.close()
        d.close()


def _stage_pair(name):
    if name == "small_pair":
        return synth.make_pair(11, 1_200_000, 3, 0.05, sv_every=60000) + (170,)
    if name == "many_long":
        return synth.make_pair(12, 8_000_000, 6, 0.05, sv_every=30000) + (170,)
    # no long triple: exact 60-base copies far apart, each too short to put more than 64 seeds in a triple
    rng = np.random.default_rng(13)
    a = rng.integers(0, 4, 300_000, dtype=np.uint8)
    b = rng.integers(0, 4, 300_001, dtype=np.uint8)
    for k in range(40):
        b[5000 + 7000 * k:5060 + 7000 * k] = a[3000 + 7100 * k:3060 + 7100 * k]
    return [a], [b], 50


def _numpy_triples(recs, layout, chain_min):
    """band segments and scanned triples of sorted records (keys of <= 64 bits): seg_start, and per segment
    its triple's end, whether it is scanned, and whether the prefilter's seed bound keeps it"""
    anti, band, jc, ic = layout[:4]
    assert not recs[:, 1].any()
    lo = recs[:, 0]
    p_band, p_jc = 12 + anti, 12 + anti + band
    up = lo >> np.uint64(p_band)
    seg = np.concatenate([[0], np.nonzero(up[1:] != up[:-1])[0] + 1]).astype(np.int64)
    ends = np.concatenate([seg[1:], [len(lo)]])
    grp = lo[seg] >> np.uint64(p_jc)
    cdiag = (lo[seg] >> np.uint64(p_band)) & np.uint64((1 << band) - 1)
    above = np.concatenate([(grp[1:] == grp[:-1]) & (cdiag[1:] == cdiag[:-1] + np.uint64(1)), [False]])
    isnew = ~np.concatenate([[False], above[:-1]])
    e = ends.copy()
    e[above] = ends[np.nonzero(above)[0] + 1]
    scanned = isnew | above
    kept = scanned & (e - seg >= (chain_min + 79) // 80)
    return seg, e, kept


@pytest.mark.parametrize("name", ["small_pair", "many_long", "no_long"])
def test_segments_work_list_and_chunk_plan_match_numpy(name):
    A, B, cm = _stage_pair(name)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    amx, bmx = int(gA.clen.max()), int(gB.clen.max())
    dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
    xA, xB = lib.DeviceGix.build(dA), lib.DeviceGix.build(dB)
    ds = lib.DeviceSeeds.find(xA, xB, amx, bmx, 10)
    xA.close()
    xB.close()
    try:
        recs = ds.download()
        layout = ds.layout + (amx, bmx)
        seg, e, kept = _numpy_triples(recs, layout, cm)
        size = e - seg
        otr, oh = ol.chains(recs, layout, 2000, cm)
        trip, hits, info = lib.chain_hits(ds, 2000, cm, chunk=CHUNK)

        # the long work triples: most seeds first, then the lower segment
        lj = np.nonzero(kept & (size > PREF_LONG))[0]
        lj = lj[np.lexsort((lj, -size[lj]))]
        nlong = info["long"]
        assert nlong == len(lj)
        assert np.array_equal(trip["start"][:nlong], seg[lj]) and np.array_equal(trip["end"][:nlong], e[lj])
        # the short ones (in the prefilter's order): the kept triples of at most 64 seeds that hold a chain
        has_chain = {int(b) for b in otr["b"][otr["nh"] > 0]}
        sj = np.nonzero(kept & (size <= PREF_LONG))[0]
        want_short = sorted(int(seg[j]) for j in sj if int(seg[j]) in has_chain)
        assert sorted(trip["start"][nlong:].tolist()) == want_short
        assert info["work"] == nlong + len(want_short)

        if name == "many_long":
            assert nlong > 256, nlong
        if name == "no_long":
            assert nlong == 0 and info["work"] > 0 and info["chunks"] == 0
        else:
            assert nlong > 0
            nch = np.maximum((size[lj] + CHUNK - 1) // CHUNK, 1)
            assert info["chunks"] == int(nch.sum())
            assert info["capacity"] == int(nch.sum()) * (HCAP + 1) + info["work"] + 16
            at = {int(b): q for q, b in enumerate(otr["b"])}
            for w in range(nlong):
                o = otr[at[int(trip["start"][w])]]
                want = oh[o["h0"]:o["h0"] + o["nh"]]
                if trip["hn"][w] & lib.CHAIN_LISTLESS:
                    assert o["nh"] > HCAP
                    continue
                got = hits[trip["h0"][w]:trip["h0"][w] + trip["hn"][w]]
                assert len(got) == len(want), w
                for f in ("alow", "ahgh", "dgmin", "dgmax"):
                    assert np.array_equal(got[f], want[f]), (w, f)

        # the band segments the extension counts
        ov = lib.DeviceOverlaps.extend(ds, dA, dB, 10, chain_min=cm)
        c = ov.counters()
        assert c["nseg"] == len(seg) and c["nwork"] == info["work"]
        ov.close()
    finally:
        ds.close()
        dA.close()
        dB.close()

"""-m gpu: SELF mode (`FastGA A`) stage by stage against the oracle.
  * the self merge (merge.cu self_merge_kernel) and the seed sort, record by record against orc_self_merge on
    the same table: every self genome the oracle is pinned on, the straddle and divergence genomes of
    self_cases.py, and its crafted tables (uploaded, so the device builds their prefix index), at freq 1, 2,
    3, 10, 64 and 255, under both seed-sort plans;
  * the extension of the straddle and divergence genomes call by call: the device's records are the oracle's
    calls that made a record, in order, and each of those is the reference's Local_Alignment with the band
    borders of a contig against itself (tests/golden/reference_runs.json); a chain across the main diagonal
    makes no call and advances the tube with 0, and the device counts it as a call."""
import os

import numpy as np
import pytest

import oracle_lib as ol
import self_cases as sc
from fastga_b200 import formats, lib
from test_oracle_pin import _self_genomes

pytestmark = pytest.mark.gpu

PINNED = ["dup", "tandem61", "tandem62", "inverted_dup", "identical_contigs", "palindrome",
          "near_diagonal_repeats", "contigs300"]
GENOMES = PINNED + sorted(sc.GENOMES)
LOW6 = np.array([~np.uint64(63), ~np.uint64(0)], dtype=np.uint64)     # the lcp field does not order seeds


def _genome(name):
    return sc.GENOMES[name]() if name in sc.GENOMES else _self_genomes()[name]


def _find_self(x, amx, freq, wide):
    old = os.environ.get("FGB_SEED_SORT_WIDE")
    os.environ["FGB_SEED_SORT_WIDE"] = "1" if wide else "0"
    try:
        return lib.DeviceSeeds.find_self(x, amx, freq)
    finally:
        if old is None:
            del os.environ["FGB_SEED_SORT_WIDE"]
        else:
            os.environ["FGB_SEED_SORT_WIDE"] = old


def _check_seeds(x, tab, pstart, amx, what):
    """find_self on x at every freq and both sort plans against orc_self_merge on (tab, pstart)"""
    for freq in sc.FREQS:
        seeds, sumlen = ol.self_merge(tab, pstart, freq)
        for wide in (False, True):
            ds = _find_self(x, amx, freq, wide)
            try:
                assert (ds.n, ds.sumlen) == (len(seeds), sumlen), (what, freq, wide)
                got = ds.download()
                want = ol.seed_records(seeds, ds.layout + (amx, amx), sort=True)
                # sorted on everything above the lcp field; seeds equal there are the same pair of posts
                assert np.array_equal(got & LOW6, want & LOW6), (what, freq, wide)
                o = np.lexsort((got[:, 0], got[:, 1]))
                assert np.array_equal(got[o], want), (what, freq, wide)
            finally:
                ds.close()


@pytest.mark.parametrize("name", GENOMES)
def test_self_seeds_match_oracle_record_by_record(name):
    g = formats.genome_from_arrays(_genome(name))
    dA = lib.DeviceGenome(g)
    x = lib.DeviceGix.build(dA)
    try:
        tab, pstart, _ = x.download()
        _check_seeds(x, tab, pstart, int(g.clen.max()), name)
    finally:
        x.close()
        dA.close()


@pytest.mark.parametrize("name", sorted(sc.TABLES))
def test_self_seeds_on_crafted_tables(name):
    T = sc.table(name)
    x = lib.DeviceGix.upload(T.tab, 4, 1 if T.ncontig <= 256 else 2, T.ncontig)
    try:
        tab, pstart, _ = x.download()
        assert np.array_equal(tab, T.tab) and np.array_equal(pstart, T.pstart())
        _check_seeds(x, T.tab, T.pstart(), sc.AMX, name)
    finally:
        x.close()


def _extend(ds, dA, g, chunk=None):
    """(records in (triple, seq) order, trace pool, counters) of fgb_extend, FGB_CHAIN_CHUNK=chunk if given"""
    old = os.environ.pop("FGB_CHAIN_CHUNK", None)
    if chunk is not None:
        os.environ["FGB_CHAIN_CHUNK"] = chunk
    try:
        ov = lib.DeviceOverlaps.extend(ds, dA, dA, g.freq)
    finally:
        os.environ.pop("FGB_CHAIN_CHUNK", None)
        if old is not None:
            os.environ["FGB_CHAIN_CHUNK"] = old
    try:
        got, pool = ov.records()
        return got, pool, ov.counters()
    finally:
        ov.close()


@pytest.mark.parametrize("name", sorted(sc.GENOMES))
def test_bordered_calls_and_straddles_call_by_call(name):
    G = sc.GENOMES[name]()
    g = formats.genome_from_arrays(G)
    dA = lib.DeviceGenome(g, want_revcomp=True)
    x = lib.DeviceGix.build(dA)
    amx = int(g.clen.max())
    ds = lib.DeviceSeeds.find_self(x, amx, 10)
    x.close()
    try:
        recs = ds.download()
        R = sc.SelfRun(G, recs, ds.layout + (amx, amx), dA.perm, straddle_zero=True)
        want = R.reference_keys(name)             # the stored keys were made from the same calls
        got, pool, cnt = _extend(ds, dA, g)
        # without chain detection: triples are scanned whole in the kernel, no hit group runs on a guessed
        # tube start (a wrong guess re-runs its triple, and its calls count again)
        got0, pool0, cnt0 = _extend(ds, dA, g, chunk="0")
    finally:
        ds.close()
        dA.close()
    made = [q for q, c in enumerate(R.calls) if c["rec"]]
    assert len(got) == len(made)
    jb, ib = R.layout[2], R.layout[3]
    for r, q in zip(got, made):
        c = R.calls[q]
        pk = int(r["pairkey"])
        assert (pk >> (jb + ib), int(R.perm[(pk >> jb) & ((1 << ib) - 1)]), int(R.perm[pk & ((1 << jb) - 1)])) == \
            (c["comp"], c["ctg1"], c["ctg2"]), q
        key = ol.path_key(r["abpos"], r["bbpos"], r["aepos"], r["bepos"], r["diffs"], r["tlen"],
                          pool[int(r["toff"]):int(r["toff"]) + int(r["tlen"])])
        assert key == ol.call_key(c) == want[q], (q, c["lbord"], c["hbord"])
    assert any(R.calls[q]["lbord"] >= 0 for q in made) and any(R.calls[q]["hbord"] >= 0 for q in made)
    # a straddle counts as a call on the device
    assert R.counters["straddles"] > 0
    assert cnt["hits"] == cnt0["hits"] == R.nhit
    assert cnt["la_calls"] >= cnt0["la_calls"] == len(R.calls) + R.counters["straddles"]
    assert len(got0) == len(got)
    for a, b in zip(got, got0):
        assert all(int(a[f]) == int(b[f]) for f in lib.OVL_DT.names if f not in ("toff", "seq"))
        assert pool[int(a["toff"]):int(a["toff"]) + int(a["tlen"])].tobytes() == \
            pool0[int(b["toff"]):int(b["toff"]) + int(b["tlen"])].tobytes()
    print(name, R.counters, "calls", len(R.calls), "records", len(got), "device calls", cnt["la_calls"],
          "without chain detection", cnt0["la_calls"])

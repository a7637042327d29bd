"""The crafted wave tubes of wave_cases.py without a GPU: the oracle's Local_Alignment calls on them equal the
reference's (stored in tests/golden/reference_runs.json, and called live where oracle/_ref is built), every
family reaches the regimes REGIMES names, and the crafted seeds are the seeds the merge would emit."""
import numpy as np
import pytest

import oracle_lib as ol
import wave_cases as wc

CASES = [(f, c) for f in wc.FAMILIES for c in wc.STRANDS]


def _id(fc):
    return "%s_%s" % (fc[0], "NC"[fc[1]])


@pytest.mark.parametrize("fc", CASES, ids=_id)
def test_oracle_calls_match_reference(fc):
    C = wc.case(*fc)
    ov, tp, nhit, calls, passes = C.run()
    want = C.reference()
    assert len(want) == len(calls) == nhit == len(C.tubes)
    assert [ol.call_key(c) for c in calls] == want
    # the records are the calls that produced one, in the same order
    rec = [c for c in calls if c["rec"]]
    assert len(rec) == len(ov)
    for c, r in zip(rec, ov):
        assert (c["abpos"], c["aepos"], c["diffs"], c["tlen"]) == (r["abpos"], r["aepos"], r["diffs"], r["tlen"])
    if ol.have_ref():
        import param_cases as pc
        live = ol.ref_local_alignments(pc.seam_calls(C.A, C.B, C.seam_jobs()), C.freq, C.ave_corr)
        assert live == want


@pytest.mark.parametrize("fc", CASES, ids=_id)
def test_family_reaches_its_regimes(fc):
    C = wc.case(*fc)
    _, _, _, calls, passes = C.run()
    got = wc.regimes_reached(calls, passes)
    assert wc.REGIMES[fc[0]] <= got, wc.REGIMES[fc[0]] - got
    # no wave fails to raise besta (see the oracle's wave()); a pass ended by a contig end with no
    # diagonal left is how a wave fails to advance
    assert not passes["stall"].any()
    for c in calls:
        if wc.call_band(passes, c) >= 252:
            assert passes["maxhop"][c["pass0"]:c["pass0"] + c["npass"]].max() > wc.WIDE_HOP
    # every pass belongs to its call, and the passes of each strand run both ways
    assert sum(c["npass"] for c in calls) == len(passes)
    assert {1, -1} <= set(passes["s"].tolist())


@pytest.mark.parametrize("fc", CASES, ids=_id)
def test_crafted_seeds_lie_on_exact_matches_and_chain_once_per_tube(fc):
    C = wc.case(*fc)
    for row in C.seeds:
        i = int(np.nonzero(C.rankA == row["icont"])[0][0])
        assert int(C.rankB[i]) == int(row["jcont"])
        x, y, Bp = wc.seed_match(row, C.A[i], C.B[i])
        p = int(row["plen"])
        assert 0 <= x and x + p <= len(C.A[i]) and 0 <= y and y + p <= len(Bp)
        assert np.array_equal(C.A[i][x:x + p], Bp[y:y + p])
    kw = {k: v for k, v in C.params.items() if k in ("chain_break", "chain_min")}
    trip, hits = ol.chains(C.recs, C.layout, **kw)
    assert len(hits) == len(C.tubes)
    keys = trip["key"][np.repeat(np.arange(len(trip)), trip["nh"])]
    assert len(set(keys.tolist())) == len(C.tubes)


@pytest.mark.parametrize("comp", wc.STRANDS)
def test_seed_builder_reproduces_merged_seeds(comp):
    """the builder, given the match positions of seeds the real merge finds on the same sequences, makes
    exactly those seeds, on both strands: x is the seed's A post, y every place of B' (B, or its reverse
    complement on strand C) that holds A[x:x+plen], found by search"""
    C = wc.case("runs", comp)
    tA, _ = ol.gix_build(C.gA, C.rankA)
    tB, sB = ol.gix_build(C.gB, C.rankB)
    seeds, _ = ol.merge(tA, tB, sB)
    rng = np.random.default_rng(5)
    same = seeds[seeds["comp"] == comp]
    assert len(same) > 1000
    sample = same[rng.choice(len(same), 500, replace=False)]
    permA, permB = C.permA, C.permB
    for s in sample:
        i, j = int(permA[s["icont"]]), int(permB[s["jcont"]])
        x, p = int(s["ipost"]), int(s["plen"])
        Bp = wc.revcomp(C.B[j]) if comp else C.B[j]
        kmer, hay = C.A[i][x:x + p].tobytes(), Bp.tobytes()
        ys, y = [], hay.find(kmer)
        while y >= 0:
            ys.append(y)
            y = hay.find(kmer, y + 1)
        rows = [wc.seed_row(comp, int(s["icont"]), int(s["jcont"]), x, y, p, len(C.B[j])) for y in ys]
        assert tuple(int(s[f]) for f in ol.SEED_DT.names) in rows

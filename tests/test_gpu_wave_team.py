"""-m gpu: the extension's wave routines as fgb_extend runs them (warp teams: front_run, wave_T, wave_P, the
interior fast path, the single-warp and wide-band fall-backs) on the crafted tubes of wave_cases.py, call by
call against the reference's Local_Alignment on the oracle's logged calls (tests/golden/reference_runs.json);
the same calls through the single-warp batch (fgb_local_alignments); and fgb_extend without chain detection."""
import os

import numpy as np
import pytest

import oracle_lib as ol
import wave_cases as wc
from fastga_b200 import lib

pytestmark = pytest.mark.gpu

CASES = [(f, c) for f in wc.FAMILIES for c in wc.STRANDS]
EXT_KW = ("chain_break", "chain_min", "align_min", "align_rate")


def _id(fc):
    return "%s_%s" % (fc[0], "NC"[fc[1]])


def _extend(C, seeds, dA, dB, chunk=None):
    """(records in (triple, seq) order, trace pool, launch number of every record, counters)"""
    old = os.environ.pop("FGB_CHAIN_CHUNK", None)
    if chunk is not None:
        os.environ["FGB_CHAIN_CHUNK"] = chunk
    try:
        ov = lib.DeviceOverlaps.extend(seeds, dA, dB, C.freq, **{k: v for k, v in C.params.items() if k in EXT_KW})
    finally:
        os.environ.pop("FGB_CHAIN_CHUNK", None)
        if old is not None:
            os.environ["FGB_CHAIN_CHUNK"] = old
    try:
        recs, pool = ov.records()
        cnt = ov.counters()
    finally:
        ov.close()
    # word 9 of a record's 40-byte header: the launch that emitted it
    launch = np.array([int(np.frombuffer(pool[int(t) - 4:int(t)].tobytes(), np.int32)[0]) for t in recs["toff"]],
                      dtype=np.int64)
    return recs, pool, launch, cnt


@pytest.mark.parametrize("fc", CASES, ids=_id)
def test_wave_team_matches_reference_call_by_call(fc):
    import torch
    C = wc.case(*fc)
    _, _, nhit, calls, passes = C.run()
    want = C.reference()
    d = torch.from_numpy(C.recs.view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    seeds = lib.seeds_from_records(d.data_ptr(), len(C.recs), C.layout[:4], C.layout[4], C.layout[5])
    del d
    dA, dB = lib.DeviceGenome(C.gA, want_revcomp=True), lib.DeviceGenome(C.gB)
    try:
        assert np.array_equal(seeds.download(), ol.seed_records(C.seeds, C.layout, sort=True))
        assert np.array_equal(dA.perm, C.permA) and np.array_equal(dB.perm, C.permB)
        recs, pool, launch, cnt = _extend(C, seeds, dA, dB)

        # records pair up one for one with the calls that produced a record: one call per tube, so the
        # (strand, contig pair) of a record names its call
        jb, ib = C.layout[2], C.layout[3]
        pk = recs["pairkey"].astype(np.int64)
        comp, ic, jc = pk >> (jb + ib), (pk >> jb) & ((1 << ib) - 1), pk & ((1 << jb) - 1)
        assert (comp == C.comp).all()
        at = {(c["ctg1"], c["ctg2"]): q for q, c in enumerate(calls)}
        got = [at[(int(C.permA[a]), int(C.permB[b]))] for a, b in zip(ic, jc)]
        assert sorted(got) == [q for q, c in enumerate(calls) if c["rec"]]
        for r, q in zip(recs, got):
            key = ol.path_key(r["abpos"], r["bbpos"], r["aepos"], r["bepos"], r["diffs"], r["tlen"],
                              pool[int(r["toff"]):int(r["toff"]) + int(r["tlen"])])
            assert key == want[q], (q, C.tubes[calls[q]["ctg1"]].note)

        # counters
        assert cnt["hits"] == nhit
        if (launch == 0).all():
            assert cnt["la_calls"] == len(calls)
        else:
            assert cnt["la_calls"] >= len(calls)

        # the device's regime: wide bands go to the wide-band launch; any other later launch is an arena
        # that grew (ST_CELLS), named here
        band = np.array([wc.call_band(passes, calls[q]) for q in got], dtype=np.int64)
        assert (launch[band > 251] >= 1).all(), [calls[q]["ctg1"] for q in np.array(got)[(band > 251) & (launch == 0)]]
        regrown = [C.tubes[calls[q]["ctg1"]].note for q in np.array(got)[(band <= 251) & (launch >= 1)]]
        print("%s: %d calls, %d records, %d from later launches, arena re-runs: %s"
              % (_id(fc), len(calls), len(recs), int((launch >= 1).sum()), regrown or "none"))
        assert not regrown
        assert cnt["paired_waves"] > 0
        # a band over 30 diagonals, or a wave that keeps no diagonal after an end clip, ends the pairing
        if any(wc.call_band(passes, c) >= 31 for c in calls) or passes["endempty"].any():
            assert cnt["paired_waves"] < cnt["waves"]

        # the same records without chain detection (triples scanned in the kernel)
        r0, p0, _, c0 = _extend(C, seeds, dA, dB, chunk="0")
        assert len(r0) == len(recs)
        for a, b in zip(recs, r0):
            assert all(int(a[f]) == int(b[f]) for f in lib.OVL_DT.names if f not in ("toff", "seq"))
            assert pool[int(a["toff"]):int(a["toff"]) + int(a["tlen"])].tobytes() == \
                p0[int(b["toff"]):int(b["toff"]) + int(b["tlen"])].tobytes()
        assert c0["hits"] == cnt["hits"]

        # the single-warp batch on the same calls
        paths, toff, traces = lib.local_alignments(dA, dB, C.seam_jobs(), C.freq,
                                                   align_rate=C.params.get("align_rate", 0.3))
        for q, p in enumerate(paths):
            assert p[6] == 0, (q, p)
            ab, bb, ae, be, df, tl = (int(v) for v in p[:6])
            assert ol.path_key(ab, bb, ae, be, df, tl, traces[int(toff[q]):int(toff[q]) + tl]) == want[q], q
    finally:
        seeds.close()
        dA.close()
        dB.close()

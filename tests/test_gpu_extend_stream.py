"""-m gpu: the extension stage on a caller's non-blocking stream.  Every copy and memset of fgb_extend is
ordered on the stream it is given, so a run on a side stream must give exactly the records and counters
of a run on the default stream, and give back every device block it took."""
import ctypes as C

import numpy as np
import pytest
import torch

from fastga_b200 import formats, lib, synth

pytestmark = pytest.mark.gpu

# counters that count work; the rest are clock cycles
COUNTS = ("hits", "la_calls", "waves", "cells", "paired_waves", "pairings", "nseg", "nwork")


def _non_blocking(stream):
    cu = C.CDLL("libcuda.so.1")
    flags = C.c_uint()
    assert cu.cuStreamGetFlags(C.c_void_p(stream.cuda_stream), C.byref(flags)) == 0
    return bool(flags.value & 1)                 # CU_STREAM_NON_BLOCKING


def _seeds(A, B):
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
    xA, xB = lib.DeviceGix.build(dA), lib.DeviceGix.build(dB)
    ds = lib.DeviceSeeds.find(xA, xB, int(gA.clen.max()), int(gB.clen.max()), 10)
    xA.close()
    xB.close()
    return gA, dA, dB, ds


def _extend(gA, dA, dB, ds, stream):
    """records (fields and trace bytes, in discovery order) and counters of one fgb_extend call"""
    ov = lib.DeviceOverlaps.extend(ds, dA, dB, gA.freq, stream=stream)
    try:
        recs, pool = ov.records()
        cnt = ov.counters()
    finally:
        ov.close()
    fields = [n for n in recs.dtype.names if n != "toff"]
    out = [tuple(int(r[n]) for n in fields) + (pool[r["toff"]:r["toff"] + r["tlen"]].tobytes(),) for r in recs]
    return out, cnt


def _same_on_side_stream(staged):
    """the records of a run on the default stream and the counters of a run on a side stream, having
    checked that the two runs agree and left no device block behind"""
    gA, dA, dB, ds = staged
    base = lib.device_live_bytes()
    want, wcnt = _extend(gA, dA, dB, ds, None)
    side = torch.cuda.Stream()
    assert _non_blocking(side)
    side.wait_stream(torch.cuda.default_stream())
    with torch.cuda.stream(side):
        got, gcnt = _extend(gA, dA, dB, ds, side.cuda_stream)
    torch.cuda.synchronize()
    assert lib.device_live_bytes() == base
    assert got == want
    assert {k: gcnt[k] for k in COUNTS} == {k: wcnt[k] for k in COUNTS}
    for h in (ds, dA, dB):
        h.close()
    return want, gcnt


def test_long_alignments_on_a_side_stream():
    # contig-long alignments: the trace staging overflows and the re-run on the wide-band kernel runs
    staged = _seeds(*synth.make_pair(13, 6_000_000, 3, 0.03, sv_every=0))
    assert staged[3].n > 0
    recs, _ = _same_on_side_stream(staged)
    assert len(recs) > 0


def test_rerun_hit_groups_on_a_side_stream(monkeypatch):
    # a cut at every hit: groups reach into their neighbours and their triples are re-run
    monkeypatch.setenv("FGB_SPEC_GAP", "0")
    staged = _seeds(*synth.make_pair(21, 3_000_000, 4, 0.08, sv_every=50_000))
    assert staged[3].n > 0
    recs, _ = _same_on_side_stream(staged)
    assert len(recs) > 0


def test_no_seeds_on_a_side_stream():
    # two short unrelated contigs: no seeds, so no work triples and no launch of the extension
    rng = np.random.default_rng(5)
    staged = _seeds([rng.integers(0, 4, 300, dtype=np.uint8)], [rng.integers(0, 4, 300, dtype=np.uint8)])
    assert staged[3].n == 0
    recs, cnt = _same_on_side_stream(staged)
    assert recs == []
    assert all(v == 0 for k, v in cnt.items() if k != "slowest_warp")
    assert all(v == 0 for v in cnt["slowest_warp"].values())

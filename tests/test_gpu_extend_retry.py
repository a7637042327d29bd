"""-m gpu: the retry ladders of the extension stage.  fgb_extend re-runs a triple whole on the wide-band
kernel when one of its items overflows an arena (pebbles ST_CELLS, trace staging ST_STAGE) and repeats a
launch whose records overflow the record buffer; fgb_local_alignments re-runs the calls that did not fit.
FGB_EXTEND_CELLS, FGB_EXTEND_STAGE and FGB_EXTEND_OUT_SLACK shrink the first sizes so that small inputs
take the steps large ones take, retry_info() proves that they did, and the records, hit counts and work
counters must be those of an unforced run, of the oracle and of the stored reference runs."""
import ctypes as C

import numpy as np
import pytest

import edge_cases
import oracle_lib as ol
import wave_cases as wc
from fastga_b200 import formats, lib, load_library, synth
from param_cases import seam_calls, seam_jobs
from test_gpu_e2e import _vs_reference

pytestmark = pytest.mark.gpu

ST_BAND, ST_CELLS, ST_STAGE = 1, 2, 3
# counters that count work; the rest are clock cycles
COUNTS = ("hits", "la_calls", "waves", "cells", "paired_waves", "pairings", "nseg", "nwork")
KNOBS = ("FGB_EXTEND_CELLS", "FGB_EXTEND_STAGE", "FGB_EXTEND_OUT_SLACK", "FGB_SPEC_GAP", "FGB_CHAIN_CHUNK")
SLACK = "1024"            # record bytes beyond the known need: every launch that adds more overflows once
CELLS = "256"             # pebbles per warp of the first launch (default 128 K; 256 K for the seam)
STAGE = "64"              # trace staging bytes per warp of the first launch (default 32 K; 64 K for the seam)


class Staged:
    """a genome pair on the device and its seeds at -f 10"""

    def __init__(self, gA, gB):
        self.gA, self.gB = gA, gB
        self.dA, self.dB = lib.DeviceGenome(self.gA, want_revcomp=True), lib.DeviceGenome(self.gB)
        xA, xB = lib.DeviceGix.build(self.dA), lib.DeviceGix.build(self.dB)
        amx, bmx = int(self.gA.clen.max()), int(self.gB.clen.max())
        self.ds = lib.DeviceSeeds.find(xA, xB, amx, bmx, 10)
        xA.close()
        xB.close()
        self.layout = self.ds.layout + (amx, bmx)
        self._oracle = None

    def oracle(self):
        """(records as _oracle_rows gives them, hits) of the oracle's search on the same seeds"""
        if self._oracle is None:
            want, wpool, whits = ol.search(self.ds.download(), self.layout, self.gA, self.gB, self.dA.perm,
                                           self.dB.perm, self.gA.freq)
            rows = [(int(r["comp"]), int(r["aread"]), int(r["bread"]), int(r["abpos"]), int(r["bbpos"]),
                     int(r["aepos"]), int(r["bepos"]), int(r["diffs"]),
                     bytes(wpool[int(r["toff"]):int(r["toff"]) + int(r["tlen"])])) for r in want]
            self._oracle = rows, whits
        return self._oracle

    def close(self):
        for h in (self.ds, self.dA, self.dB):
            h.close()


@pytest.fixture(scope="module")
def staged_small(small_pair):
    s = Staged(*small_pair)
    yield s
    s.close()


@pytest.fixture(scope="module")
def staged_gap():
    """the pair whose hit groups reach into their neighbours when cut at every hit (FGB_SPEC_GAP=0)"""
    A, B = synth.make_pair(21, 3_000_000, 4, 0.08, sv_every=50_000)
    s = Staged(formats.genome_from_arrays(A), formats.genome_from_arrays(B))
    yield s
    s.close()


def _extend(s, monkeypatch, env):
    """fgb_extend on s under the knobs env (and none other): (records in discovery order with their trace
    bytes, launch number of every record, counters, retry_info)"""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        ov = lib.DeviceOverlaps.extend(s.ds, s.dA, s.dB, s.gA.freq)
    finally:
        for k in KNOBS:
            monkeypatch.delenv(k, raising=False)
    try:
        recs, pool = ov.records()
        cnt, info = ov.counters(), ov.retry_info()
    finally:
        ov.close()
    fields = [n for n in recs.dtype.names if n != "toff"]
    rows = [tuple(int(r[n]) for n in fields) + (pool[r["toff"]:r["toff"] + r["tlen"]].tobytes(),) for r in recs]
    # word 9 of a record's 40-byte header: the launch that emitted it
    launch = [int(np.frombuffer(pool[int(t) - 4:int(t)].tobytes(), np.int32)[0]) for t in recs["toff"]]
    return rows, launch, cnt, info


def _oracle_rows(s, rows):
    """rows as the oracle gives them: (comp, A contig, B contig, abpos, bbpos, aepos, bepos, diffs, trace)"""
    jb, ib = s.layout[2], s.layout[3]
    out = []
    for r in rows:
        pk = r[2]
        out.append((pk >> (jb + ib), int(s.dA.perm[(pk >> jb) & ((1 << ib) - 1)]), int(s.dB.perm[pk & ((1 << jb) - 1)]),
                    r[3], r[4], r[5], r[6], r[7], r[9]))
    return out


MODES = {"groups": {}, "scan": {"FGB_CHAIN_CHUNK": "0"}}


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("pair", ["small_pair", "gap0"])
def test_record_buffer_regrowth_is_invisible(pair, mode, monkeypatch, request):
    """a record buffer of SLACK bytes that grows by SLACK past what each launch needed: the launches that
    overflow it are repeated, and the records and every work counter are those of an unforced run"""
    s = request.getfixturevalue("staged_small" if pair == "small_pair" else "staged_gap")
    env = dict(MODES[mode], **({"FGB_SPEC_GAP": "0"} if pair == "gap0" else {}))
    want, _, wcnt, winfo = _extend(s, monkeypatch, env)
    got, _, gcnt, ginfo = _extend(s, monkeypatch, dict(env, FGB_EXTEND_OUT_SLACK=SLACK))
    print(pair, mode, "unforced", winfo, "forced", ginfo)
    assert winfo["regrowths"] == 0
    assert ginfo["regrowths"] >= 1 and ginfo["launches"] == winfo["launches"] + ginfo["regrowths"]
    assert ginfo["reruns"] == winfo["reruns"] and ginfo["reasons"] == winfo["reasons"]
    if pair == "gap0" and mode == "groups":
        # a step repeats at most once, so two regrowths mean a re-run step overflowed as well as step 0
        assert winfo["reruns"] > 0 and ginfo["regrowths"] >= 2
    assert got == want
    assert {k: gcnt[k] for k in COUNTS} == {k: wcnt[k] for k in COUNTS}
    if pair == "small_pair":
        rows, whits = s.oracle()
        assert gcnt["hits"] == whits
        assert _oracle_rows(s, got) == rows


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("knob,reason", [("FGB_EXTEND_CELLS", ST_CELLS), ("FGB_EXTEND_STAGE", ST_STAGE)],
                         ids=["cells", "stage"])
def test_arena_ladder_gives_the_oracle_records(knob, reason, mode, staged_small, monkeypatch):
    """first arenas far too small for small_pair's alignments: items fail for that reason, their triples are
    re-run whole on larger arenas, and the records (each once, from its triple's last launch) and the hit
    count are the oracle's"""
    s = staged_small
    size = CELLS if knob == "FGB_EXTEND_CELLS" else STAGE
    got, launch, cnt, info = _extend(s, monkeypatch, dict(MODES[mode], **{knob: size}))
    print(knob, mode, info)
    assert info["reasons"] & (1 << reason)
    assert info["launches"] > 1 and info["reruns"] > 0 and info["regrowths"] == 0
    rows, whits = s.oracle()
    assert cnt["hits"] == whits
    assert _oracle_rows(s, got) == rows
    # a triple keeps the records of one launch only, its last
    last = {}
    for r, l in zip(got, launch):
        assert last.setdefault(r[0], l) == l, r[:2]


@pytest.mark.parametrize("name", ["e2e/small_pair", "e2e/long_alignments", "edge/tandem_repeats", "edge/wave_regimes"])
def test_whole_path_under_all_knobs_matches_reference(name, monkeypatch):
    """the whole path with every ladder forced (small pebble arenas, small staging, a record buffer that
    overflows at every launch) gives the stored reference run"""
    for k, v in (("FGB_EXTEND_CELLS", CELLS), ("FGB_EXTEND_STAGE", STAGE), ("FGB_EXTEND_OUT_SLACK", SLACK)):
        monkeypatch.setenv(k, v)
    if name == "e2e/small_pair":
        _vs_reference("small_pair", 11, 1_200_000, 3, 0.05, 60_000)
    elif name == "e2e/long_alignments":
        _vs_reference("long_alignments", 13, 6_000_000, 3, 0.03, 0)
    else:
        case = name.split("/")[1]
        A, B, _, check = edge_cases.CASES[case]()
        st = edge_cases.reference_run(case)
        alns, stats = lib.fastga(formats.genome_from_arrays(A), formats.genome_from_arrays(B))
        assert stats["nseeds"] == st["seeds"] and stats["nhits"] == st["hits"]
        assert alns.nraw == st["alns"] and len(alns) == st["kept"] == st["records"]
        assert ol.md5_lines(alns.canonical_lines()) == st["aln_md5"]
        check(alns, stats["nhits"])


def test_long_alignments_retry_regime(monkeypatch):
    """what the default sizes do on the contig-long alignments of the long_alignments pair: the trace
    staging overflows, never the pebble arena, and the triples are re-run"""
    A, B = synth.make_pair(13, 6_000_000, 3, 0.03, sv_every=0)
    s = Staged(formats.genome_from_arrays(A), formats.genome_from_arrays(B))
    try:
        rows, launch, cnt, info = _extend(s, monkeypatch, {})
    finally:
        s.close()
    print("long_alignments:", info, "records", len(rows), "launches of the records", sorted(set(launch)))
    # contig-long traces overflow the trace staging (32 KB a warp); the pebble arenas hold
    assert info["reasons"] == 1 << ST_STAGE
    assert info["launches"] > 1 and info["reruns"] > 0 and info["regrowths"] == 0
    assert len(rows) > 0 and max(launch) > 0


# ---------------------------------------------------------------------------------------------
#  fgb_local_alignments
# ---------------------------------------------------------------------------------------------

SEAM = ["batch", "batch_borders"] + ["%s_%s" % (f, "NC"[c]) for f in wc.FAMILIES for c in wc.STRANDS]


def _seam(name):
    """(genome A, genome B, jobs, align_rate, path_key of the reference for every job)"""
    if name.startswith("batch"):
        borders = name == "batch_borders"
        A, B, jobs = seam_jobs(41 + int(borders), borders)
        gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
        calls = seam_calls(A, B, jobs)
        want = ol.reference("local_alignment/" + name, ol.digest(calls, gA.freq),
                            lambda: ol.ref_local_alignments(calls, gA.freq))
        return gA, gB, np.ascontiguousarray(jobs, dtype=np.int32).reshape(-1, 8), 0.3, want
    f, c = name.rsplit("_", 1)
    Cs = wc.case(f, "NC".index(c))
    return Cs.gA, Cs.gB, Cs.seam_jobs(), Cs.params.get("align_rate", 0.3), Cs.reference()


def _keys(paths, toff, traces):
    out = []
    for q, p in enumerate(paths):
        assert p[6] == 0, (q, p)
        ab, bb, ae, be, df, tl = (int(v) for v in p[:6])
        out.append(ol.path_key(ab, bb, ae, be, df, tl, traces[int(toff[q]):int(toff[q]) + tl]))
    return out


def _raw_local_alignments(dA, dB, jobs, freq, align_rate, traces_cap):
    """fgb_local_alignments once: (return code, *traces_used)"""
    tables, ave = lib.align_spec(1.0 - align_rate, freq)
    n = jobs.shape[0]
    paths = np.zeros((n, 7), dtype=np.int32)
    toff = np.zeros(n, dtype=np.int64)
    traces = np.zeros(max(traces_cap, 1), dtype=np.uint8)
    used = C.c_longlong()
    L = load_library()
    rc = L.fgb_local_alignments(dA.h, dB.h, n, jobs.ctypes.data, tables.ctypes.data, ave, 100, paths.ctypes.data,
                                toff.ctypes.data, traces.ctypes.data, traces_cap, C.byref(used), None)
    return rc, used.value


def record_overflow_jobs(paths):
    """the jobs whose records (40-byte header + trace padded to 8 bytes) exceed the 256 bytes a job is
    given in fgb_local_alignments' record buffer by more than 64: with FGB_EXTEND_OUT_SLACK=64 and no
    trace buffer, their records overflow it"""
    return np.nonzero(paths[:, 5] >= 300)[0]


@pytest.mark.parametrize("name", SEAM)
def test_local_alignments_ladder_matches_reference(name, monkeypatch):
    gA, gB, jobs, rate, want = _seam(name)
    dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
    try:
        # small arenas: the calls that outgrow them are re-run on larger ones, up to four rounds
        monkeypatch.setenv("FGB_EXTEND_CELLS", "4096")
        monkeypatch.setenv("FGB_EXTEND_STAGE", "256")
        paths, toff, traces = lib.local_alignments(dA, dB, jobs, gA.freq, align_rate=rate)
        assert _keys(paths, toff, traces) == want
        monkeypatch.delenv("FGB_EXTEND_CELLS")
        monkeypatch.delenv("FGB_EXTEND_STAGE")
        # a record buffer too small for the records: FGB_ERR_OVERFLOW with at least the trace bytes needed
        sel = record_overflow_jobs(paths)
        assert len(sel) > 0 or not name.startswith("batch")
        if len(sel) == 0:
            return
        sub = np.ascontiguousarray(jobs[sel])
        need = int(paths[sel, 5].sum())
        monkeypatch.setenv("FGB_EXTEND_OUT_SLACK", "64")
        rc, used = _raw_local_alignments(dA, dB, sub, gA.freq, rate, 0)
        assert rc == -4 and used >= need, (rc, used, need)
        p2, t2, tr2 = lib.local_alignments(dA, dB, sub, gA.freq, align_rate=rate)
        assert _keys(p2, t2, tr2) == [want[q] for q in sel]
    finally:
        dA.close()
        dB.close()


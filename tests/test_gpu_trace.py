"""-m gpu: trace points -> edit scripts (fgb_compute_trace_pts, SURVEY row a-17) against the
UNMODIFIED reference's Compute_Trace_PTS (oracle/_ref/libfastga_ref.so; its results stored in
tests/golden/reference_runs.json) on the alignments the path emits: same int script, same diffs,
for every record."""
import ctypes as C
import hashlib

import numpy as np
import pytest

import edge_cases
import oracle_lib as ol
from fastga_b200 import formats, lib, synth

pytestmark = pytest.mark.gpu


def _aln_key(alns, i):
    return hashlib.md5(alns.fields[i].astype(np.int32).tobytes() + alns.trace(i).tobytes()).hexdigest()[:12]


def _script_key(script, diffs):
    return hashlib.md5(np.asarray(script, dtype=np.int32).tobytes() + b"%d" % diffs).hexdigest()[:12]


def _reference_scripts(gA, gB, alns, limit=None):
    """Compute_Trace_PTS(aln, work, 100, GREEDIEST, 1, -1) as ALNtoPAF.c:251-272 calls it"""
    ref = C.CDLL(ol.REF_SO)
    ref.New_Work_Data.restype = C.c_void_p
    ref.Compute_Trace_PTS.argtypes = [C.POINTER(ol.Alignment), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    work = ref.New_Work_Data()
    A = [ol._framed(gA.contig(c)) for c in range(gA.ncontig)]
    B = [ol._framed(gB.contig(c)) for c in range(gB.ncontig)]
    BC = [ol._framed(3 - gB.contig(c)[::-1]) for c in range(gB.ncontig)]
    out = []
    n = len(alns) if limit is None else min(limit, len(alns))
    for i in range(n):
        comp, ar, br, ab, bb, ae, be, df, tl = (int(x) for x in alns.fields[i])
        pts = alns.trace(i).astype(np.uint16)            # Decompress_TraceTo16
        p = ol.Path(pts.ctypes.data, tl, df, ab, bb, ae, be)
        a, b = A[ar], (BC[br] if comp else B[br])
        al = ol.Alignment(C.pointer(p), 2 if comp else 0, a.ctypes.data + 1, b.ctypes.data + 1, len(a) - 2, len(b) - 2)
        assert ref.Compute_Trace_PTS(C.byref(al), work, 100, 0, 1, -1) == 0
        sc = np.ctypeslib.as_array(C.cast(p.trace, C.POINTER(C.c_int32)), shape=(max(p.tlen, 1),))[:p.tlen].copy()
        out.append((sc, p.diffs))
    return out


def _check_pair(name, seed, total, ncontig, div, sv, flip=()):
    A, B = synth.make_pair(seed, total, ncontig, div, sv_every=sv)
    for i in flip:                                   # whole contigs on the opposite strand
        B[i] = (3 - B[i][::-1]).astype(np.uint8)
    return _check_contigs(name, A, B)


def reference_scripts(name, A, B):
    """the reference's script key of every record the path must emit on A, B: the oracle's records,
    which the e2e tests pin bit-exactly"""
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)

    def run():
        ralns = ol.oracle_pipeline(gA, gB)["alns"]
        return {_aln_key(ralns, i): _script_key(sc, df)
                for i, (sc, df) in enumerate(_reference_scripts(gA, gB, ralns))}
    return ol.reference("trace_pts/" + name, ol.digest(A, B), run)


def _check_contigs(name, A, B):
    want = reference_scripts(name, A, B)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    alns, _ = lib.fastga(gA, gB)
    assert len(alns) > 0 and len(alns) == len(want)
    dA, dB = lib.DeviceGenome(gA), lib.DeviceGenome(gB, want_revcomp=True)
    soff, script, diffs = lib.compute_trace_pts(dA, dB, alns)
    assert (diffs >= 0).all()
    ncomp = 0
    for i in range(len(alns)):
        got = script[soff[i]:soff[i + 1]]
        assert _script_key(got, int(diffs[i])) == want[_aln_key(alns, i)], (i, got[:8], int(diffs[i]))
        ncomp += int(alns.fields[i, 0])
    return len(alns), ncomp, alns


def test_scripts_match_reference_5pct():
    n, ncomp, _ = _check_pair("5pct", 21, 3_000_000, 4, 0.05, 60_000)
    assert n > 10


def test_scripts_match_reference_15pct_both_strands():
    n, ncomp, _ = _check_pair("15pct_both_strands", 22, 2_000_000, 5, 0.15, 30_000, flip=(0, 3))
    assert n > 10 and ncomp > 0


def test_scripts_match_reference_past_2_24():
    """the long_contigs pair of tests/edge_cases.py: alignments at coordinates >= 2^24 on both strands"""
    A, B, _, _ = edge_cases.long_contigs()
    n, ncomp, alns = _check_contigs("long_contigs", A, B)
    past = alns.fields[:, 5] > (1 << 24)
    assert past.any() and 0 < int(alns.fields[past, 0].sum()) < int(past.sum())


def test_inconsistent_trace_points_are_flagged_not_fatal():
    A, B = synth.make_pair(23, 600_000, 2, 0.05, sv_every=50_000)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    alns, _ = lib.fastga(gA, gB)
    dA, dB = lib.DeviceGenome(gA), lib.DeviceGenome(gB, want_revcomp=True)
    i = int(np.argmax(alns.fields[:, 8]))
    alns.pool[int(alns.toff[i]) + 2] = 0          # claim zero differences in a tile that has some
    alns.pool[int(alns.toff[i]) + 4] = 0
    alns.pool[int(alns.toff[i]) + 6] = 0
    soff, script, diffs = lib.compute_trace_pts(dA, dB, alns)
    good = [k for k in range(len(alns)) if k != i]
    assert (diffs[good] >= 0).all()
    assert diffs[i] == -1 or diffs[i] >= 0        # only flagged when a tile really cannot be aligned

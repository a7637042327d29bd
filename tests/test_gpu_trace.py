"""-m gpu: trace points -> edit scripts (fgb_compute_trace_pts, SURVEY row a-17) against the
UNMODIFIED reference's Compute_Trace_PTS (oracle/_ref/libfastga_ref.so; its results stored in
tests/golden/reference_runs.json) on the alignments the path emits: same int script, same diffs,
for every record."""
import hashlib

import numpy as np
import pytest

import edge_cases
import oracle_lib as ol
from fastga_b200 import formats, lib, synth

pytestmark = pytest.mark.gpu


def _aln_key(alns, i):
    return hashlib.md5(alns.fields[i].astype(np.int32).tobytes() + alns.trace(i).tobytes()).hexdigest()[:12]


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
        return {_aln_key(ralns, i): key for i, key in enumerate(ol.ref_trace_pts(ralns, gA, gB))}
    return ol.reference("trace_pts/" + name, ol.digest(A, B), run)


def _check_contigs(name, A, B):
    want = reference_scripts(name, A, B)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    alns, _ = lib.fastga(gA, gB)
    assert len(alns) > 0 and len(alns) == len(want)
    dA, dB = lib.DeviceGenome(gA), lib.DeviceGenome(gB, want_revcomp=True)
    soff, script, diffs, bad = lib.compute_trace_pts(dA, dB, alns, with_bad=True)
    assert (diffs >= 0).all() and bad == 0
    ncomp = 0
    for i in range(len(alns)):
        got = script[soff[i]:soff[i + 1]]
        assert ol.script_key(got, int(diffs[i])) == want[_aln_key(alns, i)], (i, got[:8], int(diffs[i]))
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


def _understate(alns):
    """the longest record with zero differences claimed for three of its tiles that have some"""
    i = int(np.argmax(alns.fields[:, 8]))
    for k in (2, 4, 6):
        alns.pool[int(alns.toff[i]) + k] = 0
    return i


def test_inconsistent_trace_points_are_flagged_not_fatal():
    """Understated tile counts do not make a record bad by themselves: the reference gives every tile
    the record's largest count as its wave limit (align.c:6210-6221), so it still computes this
    record's script, and so must the device."""
    A, B = synth.make_pair(23, 600_000, 2, 0.05, sv_every=50_000)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)

    def run():
        ralns = ol.oracle_pipeline(gA, gB)["alns"]
        i = _understate(ralns)
        return dict(record=_aln_key(ralns, i), script=ol.ref_trace_pts(ralns, gA, gB)[i])
    want = ol.reference("trace_pts/understated_tiles", ol.digest(A, B), run)
    assert want["script"] != "fail"
    alns, _ = lib.fastga(gA, gB)
    i = _understate(alns)
    assert _aln_key(alns, i) == want["record"]
    dA, dB = lib.DeviceGenome(gA), lib.DeviceGenome(gB, want_revcomp=True)
    soff, script, diffs, bad = lib.compute_trace_pts(dA, dB, alns, with_bad=True)
    assert bad == 0 and (diffs >= 0).all()
    assert ol.script_key(script[soff[i]:soff[i + 1]], int(diffs[i])) == want["script"]

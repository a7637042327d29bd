"""-m gpu: the align.h seam -- fgb_local_alignments (batched Local_Alignment) against the UNMODIFIED
reference's Local_Alignment (oracle/_ref/libfastga_ref.so; its results stored in
tests/golden/reference_runs.json) on random call tuples, borders included."""
import pytest

import oracle_lib as ol
from fastga_b200 import formats, lib
from param_cases import seam_calls, seam_jobs

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("borders", [False, True])
def test_batched_local_alignment_matches_reference(borders):
    A, B, jobs = seam_jobs(41 + int(borders), borders)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    calls = seam_calls(A, B, jobs)
    want = ol.reference("local_alignment/batch%s" % ("_borders" if borders else ""), ol.digest(calls, gA.freq),
                        lambda: ol.ref_local_alignments(calls, gA.freq))
    dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
    paths, toff, traces = lib.local_alignments(dA, dB, jobs, gA.freq)
    nonempty = 0
    for q, got in enumerate(paths):
        assert got[6] == 0, (q, got)
        ab, bb, ae, be, df, tl = (int(v) for v in got[:6])
        assert ol.path_key(ab, bb, ae, be, df, tl, traces[int(toff[q]):int(toff[q]) + tl]) == want[q], (q, jobs[q], got)
        nonempty += int(ae > ab)
    assert nonempty > 100

"""-m gpu: trace_tiles_kernel (fgb_compute_trace_pts) on the crafted records of tests/trace_cases.py.
Every record's output must equal what the unmodified reference's Compute_Trace_PTS computed on it
(tests/golden/reference_runs.json: the script key, or "fail" where the kernel must answer -1), and
pass the independent checks of trace_cases: the script replays to its diffs, the diffs are the sum
of the tiles' edit distances, and a record is bad exactly when a tile needs more waves than the
record's wave limit."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import oracle_lib as ol
import trace_cases as tc
from fastga_b200 import formats, lib

pytestmark = pytest.mark.gpu

NAMES = sorted(tc.CASES)


def _run(c, stream=None):
    gA, gB = c.genomes()
    dA, dB = lib.DeviceGenome(gA), lib.DeviceGenome(gB, want_revcomp=True)
    try:
        return lib.compute_trace_pts(dA, dB, c.alns(), stream=stream, with_bad=True)
    finally:
        dA.close()
        dB.close()


def _keys(soff, script, diffs):
    return ["fail" if diffs[k] == -1 else ol.script_key(script[soff[k]:soff[k + 1]], int(diffs[k]))
            for k in range(len(diffs))]


@pytest.mark.parametrize("name", NAMES)
def test_scripts_match_reference_and_independent_checks(name):
    c = tc.case(name)
    want = tc.reference_run(name)
    t0 = time.perf_counter()
    soff, script, diffs, bad = _run(c)
    secs = time.perf_counter() - t0
    got = _keys(soff, script, diffs)
    assert len(got) == len(want)
    wrong = [k for k in range(len(got)) if got[k] != want[k]]
    assert not wrong, (name, len(wrong), [(k, got[k], want[k], c.fields[k].tolist()) for k in wrong[:5]])
    assert bad == int((diffs == -1).sum())
    expect = tc.expect_bad(c)
    assert list(diffs == -1) == list(expect)
    eds = tc.tile_eds(c)
    for k in range(len(diffs)):
        if expect[k]:
            assert soff[k] == soff[k + 1]
        else:
            tc.check_script(script[soff[k]:soff[k + 1]], int(diffs[k]), c.fields[k], c.trace(k), c.aseq(k),
                            c.bseq(k), eds[k])
    print("%s: %d records, %d bad, %.3f s" % (name, len(diffs), bad, secs))


def test_self_records_are_the_paths():
    """self_records holds the oracle's SELF records of its genome; the device path emits the same"""
    c = tc.case("self_records")
    alns, _ = lib.fastga_self(formats.genome_from_arrays(c.A))
    assert alns.canonical_lines() == c.alns().canonical_lines()


def _non_blocking(stream):
    cu = C.CDLL("libcuda.so.1")
    flags = C.c_uint()
    assert cu.cuStreamGetFlags(C.c_void_p(stream.cuda_stream), C.byref(flags)) == 0
    return bool(flags.value & 1)                 # CU_STREAM_NON_BLOCKING


def test_side_stream_gives_identical_output():
    """records with understated tiles (the second launch) on a non-blocking stream: the same output,
    and every device block given back"""
    c = tc.case("recorded_diffs")
    base = lib.device_live_bytes()
    want = _run(c)
    side = torch.cuda.Stream()
    assert _non_blocking(side)
    side.wait_stream(torch.cuda.default_stream())
    with torch.cuda.stream(side):
        got = _run(c, side.cuda_stream)
    torch.cuda.synchronize()
    assert lib.device_live_bytes() == base
    for g, w in zip(got[:3], want[:3]):
        assert np.array_equal(g, w)
    assert got[3] == want[3] and want[3] > 0


def test_tile_wider_than_int16_is_refused():
    """furthest points are int16: a tile of 32767 bases runs, one of 32768 is refused before anything
    is allocated"""
    rng = np.random.default_rng(9)
    for m, ok in ((32767, True), (32768, False)):
        bd = tc.Builder(int(rng.integers(1 << 30)))
        k = bd.path(m, np.zeros(m, np.int8), 0.0, 0, pre=(5, 5), post=(5, 5))
        bd.rows[k][8] = 0
        bd.traces[k] = bd.traces[k][:0]
        c = bd.case()
        base = lib.device_live_bytes()
        if ok:
            soff, script, diffs, bad = _run(c)
            assert list(diffs) == [0] and bad == 0 and len(script) == 0
        else:
            with pytest.raises(lib.FgbError, match=r"\(-3\)"):
                _run(c)
        assert lib.device_live_bytes() == base

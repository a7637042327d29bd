"""CPU pins at non-default FastGA parameters (-c -s -l -i -f) and on skewed base composition:
  * the alignment spec tables (trim table, score table, ave_path) of the library's host function and of
    the oracle against the reference's New_Align_Spec, across -i and across every base-bias step;
  * the oracle's Local_Alignment against the reference's at other identities and a skewed composition,
    including the job batches the GPU seam test runs (tests/test_gpu_params.py);
  * the whole path through the oracle against `FastGA <flags>` for every case of tests/param_cases.py,
    pair and SELF mode.
The reference's results are stored in tests/golden/reference_runs.json (oracle_lib.reference), so the GPU
tests compare against the same records."""
import ctypes as C
import hashlib

import numpy as np
import pytest

import oracle_lib as ol
import param_cases as pc
from fastga_b200 import formats, lib
from test_oracle_pin import _la_check_oracle, _la_compare, _self_genomes

# ---------------------------------------------------------------------------------------------
#  New_Align_Spec
# ---------------------------------------------------------------------------------------------

I_TEXTS = ["0.55", "0.6", "0.65", "0.7", "0.75", "0.8", "0.85", "0.9", "0.95", "0.99"]
BIAS_STEPS = [0.175 + 0.05 * k for k in range(7)]           # match where (match+.025)*20 is whole


def _vec(half):
    """float32 frequencies with A = T = half, C = G splitting the rest"""
    h = np.float32(half)
    g = np.float32((1.0 - 2.0 * float(h)) / 2)
    return np.array([h, g, g, h], np.float32)


def _ulps(x, d):
    x = np.float32(x)
    for _ in range(abs(d)):
        x = np.nextafter(x, np.float32(np.inf if d > 0 else -np.inf), dtype=np.float32)
    return x


def _spec_freqs():
    """A+T within two float32 ulps either side of every bias step and of the .2 cap, the same mirrored
    (A+T > .5), far below the cap, all zero (the cap again), NaN (the 'undefined' case, match = .5) and
    uniform"""
    out = []
    for s in BIAS_STEPS + [0.2]:
        for m in (s, 1.0 - s):
            for d in (-2, -1, 0, 1, 2):
                out.append(_vec(_ulps(m / 2, d)))
    for at in (0.0, 0.01, 0.02, 0.03, 0.1, 0.3, 0.7, 0.9, 0.97, 0.99, 1.0):
        out.append(_vec(at / 2))
    out.append(np.zeros(4, np.float32))
    out.append(np.full(4, np.nan, np.float32))
    out.append(np.full(4, 0.25, np.float32))
    return out


def _raw_bias(f):
    """New_Align_Spec's bias index before the 80/20 cap (float sum, double arithmetic, align.c:240-249)"""
    match = float(np.float32(f[0]) + np.float32(f[3]))
    if (match <= 0.) == (match > 0.):
        match = .5
    if match > .5:
        match = 1. - match
    return int((match + .025) * 20. - 1.), match


def test_spec_grid_straddles_every_bias_step():
    """each step of the grid really has frequency vectors on both sides, in the reference's arithmetic"""
    F = _spec_freqs()
    for k, s in enumerate(BIAS_STEPS + [0.2]):
        for side in range(2):
            near = F[(2 * k + side) * 5:(2 * k + side + 1) * 5]
            raw = {_raw_bias(f)[0] for f in near}
            below = {_raw_bias(f)[1] < 0.2 for f in near}
            assert len(raw) == 2 or len(below) == 2, (s, side, raw)
    assert {3 if _raw_bias(f)[1] < .2 else _raw_bias(f)[0] for f in F} == set(range(3, 10))
    assert {_raw_bias(f)[0] for f in F} >= {0, 1, 2}           # indices the cap replaces


class RefSpec(C.Structure):                  # _Align_Spec, align.c:183-191
    _fields_ = [("ave_corr", C.c_double), ("trace_space", C.c_int), ("reach", C.c_int), ("freq", C.c_float * 4),
                ("ave_path", C.c_int), ("score", C.POINTER(C.c_int16)), ("table", C.POINTER(C.c_int16))]


def _md5(tables):
    return hashlib.md5(np.ascontiguousarray(tables, dtype=np.int16).tobytes()).hexdigest()


def _ref_specs(ave_corr, freqs):
    """[md5 of score[32768] + table[32768], ave_path] of the reference's New_Align_Spec per vector"""
    ref = C.CDLL(ol.REF_SO)
    ref.New_Align_Spec.restype = C.POINTER(RefSpec)
    ref.New_Align_Spec.argtypes = [C.c_double, C.c_int, C.POINTER(C.c_float), C.c_int]
    ref.Free_Align_Spec.argtypes = [C.POINTER(RefSpec)]
    out = []
    for f in freqs:
        sp = ref.New_Align_Spec(ave_corr, 100, (C.c_float * 4)(*[float(v) for v in f]), 0)
        s = np.ctypeslib.as_array(sp.contents.score, shape=(32768,))
        t = np.ctypeslib.as_array(sp.contents.table, shape=(32768,))
        out.append([_md5(np.concatenate([s, t])), int(sp.contents.ave_path)])
        ref.Free_Align_Spec(sp)
    return out


@pytest.mark.parametrize("i_text", I_TEXTS)
def test_align_spec_tables_match_reference(i_text):
    """fgb_align_spec (the library's host function) and the oracle build the reference's trim and score
    tables and ave_path, bit for bit, at -i<i_text> for every frequency vector of the grid"""
    ac = pc.ave_corr(i_text)
    freqs = _spec_freqs()
    want = ol.reference("spec/i" + i_text, ol.digest(ac, freqs), lambda: _ref_specs(ac, freqs))
    assert len({w[0] for w in want}) > 1
    for f, (md5, ave) in zip(freqs, want):
        tabs, lave = lib.align_spec(ac, f)
        assert (_md5(tabs), lave) == (md5, ave), (i_text, f.tolist())
        _, otabs, oave = ol.make_spec(f, ac)
        assert (_md5(otabs), oave) == (md5, ave), (i_text, f.tolist())


def test_align_spec_ave_path_at_documented_rates():
    """ave_path for uniform composition: 54 at -i.9, 33 at -i.55, 42 at the default"""
    u = np.full(4, 0.25, np.float32)
    assert [lib.align_spec(pc.ave_corr(i), u)[1] for i in ("0.9", "0.55", "0.7")] == [54, 33, 42]


# ---------------------------------------------------------------------------------------------
#  Local_Alignment at other identities and compositions
# ---------------------------------------------------------------------------------------------

SKEWED = np.array([.15, .35, .35, .15], np.float32)          # A+T = .3: bias index 5


@pytest.mark.parametrize("seed,borders", [(1, False), (11, True)])
@pytest.mark.parametrize("i_text", ["0.55", "0.8", "0.95"])
def test_local_alignment_at_identity_vs_reference_library(i_text, seed, borders):
    _la_compare(seed, borders, ave_corr=pc.ave_corr(i_text))


@pytest.mark.parametrize("seed,borders", [(1, False), (11, True)])
def test_local_alignment_skewed_composition_vs_reference_library(seed, borders):
    assert ol.make_spec(SKEWED)[2] == int(60 * (1 - .850 * .3))
    _la_compare(seed, borders, freq=SKEWED)


@pytest.mark.parametrize("name", sorted(pc.SEAM_CASES))
def test_seam_batches_oracle_vs_reference(name):
    """the job batches of the GPU seam test at other identities: records the reference and pins the oracle"""
    _, _, _, calls, freq, i_text = pc.seam_case(name)
    want = pc.seam_reference(name, calls, freq, i_text)
    _la_check_oracle(calls, want, freq, pc.ave_corr(i_text))


# ---------------------------------------------------------------------------------------------
#  the whole path
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(pc.CASES))
def test_oracle_at_parameters_vs_reference(name):
    flags, A, B = pc.case(name)
    st = pc.reference_run(name, A, B)
    r = ol.oracle_pipeline(formats.genome_from_arrays(A), formats.genome_from_arrays(B), **pc.params(flags))
    assert (r["nseeds"], r["nhit"], r["nraw"], len(r["lines"])) == \
        (st.get("seeds", 0), st["hits"], st["alns"], st["kept"])
    assert r["nchain"] == r["nhit"]
    assert len(r["lines"]) == st["records"] and ol.md5_lines(r["lines"]) == st["aln_md5"]
    ol.check_filters_and_order(r, st)
    assert st["records"] >= 5


def test_oracle_self_mode_at_parameters_vs_reference():
    G = _self_genomes()[pc.SELF_NAME]
    st = pc.self_reference_run(G)
    r = ol.oracle_pipeline_self(formats.genome_from_arrays(G), **pc.params(pc.SELF_FLAGS))
    # every thread of the reference halves its own pair count (FastGA.c:1907): off by < #threads
    assert abs(r["nseeds"] // 2 - st["seeds"]) < pc.SELF_THREADS
    assert r["nhit"] == st["hits"] and r["nraw"] == st["alns"]
    assert len(r["lines"]) == st["records"] and ol.md5_lines(r["lines"]) == st["aln_md5"]
    ol.check_filters_and_order(r, st)
    assert st["records"] > 10

"""-m gpu: the CUDA path at non-default FastGA parameters (-c -s -l -i -f) and on skewed base composition,
against the reference's stored results for the cases of tests/param_cases.py (recorded, and pinned to the
oracle, by tests/test_params.py), plus the compiled drop-in against the stock binary at non-default flags."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle_lib as ol
import param_cases as pc
from fastga_b200 import formats, lib, synth
from test_oracle_pin import _self_genomes

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(pc.CASES))
def test_fastga_at_parameters_vs_reference(name):
    flags, A, B = pc.case(name)
    st = pc.reference_run(name, A, B)
    alns, stats = lib.fastga(formats.genome_from_arrays(A), formats.genome_from_arrays(B), **pc.params(flags))
    assert stats["nseeds"] == st.get("seeds", 0)
    assert stats["nhits"] == st["hits"]
    assert alns.nraw == st["alns"]
    assert len(alns) == st["kept"] == st["records"]
    assert ol.md5_lines(alns.canonical_lines()) == st["aln_md5"]


def test_self_mode_at_parameters_vs_oracle():
    g = formats.genome_from_arrays(_self_genomes()[pc.SELF_NAME])
    p = pc.params(pc.SELF_FLAGS)
    want = ol.oracle_pipeline_self(g, **p)
    alns, stats = lib.fastga_self(g, **p)
    assert stats["nseeds"] == want["nseeds"]
    assert stats["nhits"] == want["nhit"]
    assert alns.nraw == want["nraw"]
    assert alns.canonical_lines() == want["lines"]
    assert len(alns) > 10


@pytest.mark.parametrize("name", sorted(pc.SEAM_CASES))
def test_batched_local_alignment_at_identity_vs_reference(name):
    A, B, jobs, calls, freq, i_text = pc.seam_case(name)
    want = pc.seam_reference(name, calls, freq, i_text)
    dA, dB = lib.DeviceGenome(formats.genome_from_arrays(A), want_revcomp=True), \
        lib.DeviceGenome(formats.genome_from_arrays(B))
    paths, toff, traces = lib.local_alignments(dA, dB, jobs, freq, align_rate=pc.params(["-i" + i_text])["align_rate"])
    nonempty = 0
    for q, got in enumerate(paths):
        assert got[6] == 0, (q, got)
        ab, bb, ae, be, df, tl = (int(v) for v in got[:6])
        assert ol.path_key(ab, bb, ae, be, df, tl, traces[int(toff[q]):int(toff[q]) + tl]) == want[q], (q, jobs[q], got)
        nonempty += int(ae > ab)
    assert nonempty > 100


def test_local_alignment_band_wider_than_shared_state():
    """call 3 of the -i.55 batch: its band outgrows the shared-memory wave state, and the batch used to
    return it with status 1 and an empty path instead of re-running it on the wide-band kernel"""
    A, B, jobs, calls, freq, i_text = pc.seam_case("i0.55")
    want = pc.seam_reference("i0.55", calls, freq, i_text)
    dA, dB = lib.DeviceGenome(formats.genome_from_arrays(A), want_revcomp=True), \
        lib.DeviceGenome(formats.genome_from_arrays(B))
    paths, toff, traces = lib.local_alignments(dA, dB, jobs[3:4], freq,
                                              align_rate=pc.params(["-i" + i_text])["align_rate"])
    ab, bb, ae, be, df, tl, status = (int(v) for v in paths[0])
    assert status == 0 and ae > ab
    assert ol.path_key(ab, bb, ae, be, df, tl, traces[:tl]) == want[3]


@pytest.mark.parametrize("name", ["at_rich", "gc_rich"])
def test_gix_build_on_skewed_composition_matches_oracle(name):
    """k-mer tables of low-complexity-prone genomes: the syncmer tie rule on runs of equal minimizers"""
    _, A, B = pc.case(name)
    for contigs in (A, B):
        g = formats.genome_from_arrays(contigs)
        dg = lib.DeviceGenome(g)
        perm, rank = ol.contig_rank(g.clen)
        assert np.array_equal(dg.perm, perm)
        want, wstart = ol.gix_build(g, rank)
        tab, pstart, _ = lib.DeviceGix.build(dg).download()
        assert np.array_equal(tab, want)
        assert np.array_equal(pstart, wstart)


DROPIN = os.path.join(ol.REF_DIR, "b200", "FastGA")
DROPIN_FLAGS = ["-f20", "-c60", "-s800", "-l300", "-i.8"]


def _run(binary, args, wd):
    r = subprocess.run([binary] + args, cwd=wd, env=ol.ref_env(), stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stderr


@pytest.mark.skipif(not (ol.have_ref() and os.path.exists(DROPIN)), reason="oracle/_ref/b200/FastGA not built")
def test_dropin_flags_reach_the_library():
    """the drop-in hands FastGA's parsed options to the library as the reference uses them (-c and -s doubled,
    -i as 1-i): same records and -v counters as the stock binary at non-default flags"""
    with tempfile.TemporaryDirectory() as wd:
        A, B = synth.make_pair(33, 1_500_000, 3, 0.1, sv_every=40_000)
        formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", 1))
        formats.write_fasta(os.path.join(wd, "B.fasta"), synth.scaffolds_of(B, "sb", 1))
        log_ref = _run(os.path.join(ol.REF_DIR, "FastGA"), ["-v", "-k", "-T8", "-P" + wd, "-1:ref"] + DROPIN_FLAGS +
                       ["A", "B"], wd)
        log_b200 = _run(DROPIN, ["-v", "-T8", "-P" + wd, "-1:b200"] + DROPIN_FLAGS + ["A", "B"], wd)
        ref = ol.oneview_records(os.path.join(wd, "ref.1aln"))
        assert len(ref) > 10 and ol.oneview_records(os.path.join(wd, "b200.1aln")) == ref
        a, b = ol.parse_fastga_log(log_ref), ol.parse_fastga_log(log_b200)
        assert (a["seeds"], a["hits"], a["alns"], a["kept"]) == (b["seeds"], b["hits"], b["alns"], b["kept"])

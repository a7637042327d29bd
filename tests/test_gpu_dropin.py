"""-m gpu: the COMPILED drop-in -- the reference's own FastGA.c with integration/FastGA_b200.patch,
linked against libfastga_b200.so (oracle/_ref/b200/FastGA, built by `make -f oracle/Makefile.ref dropin`)
-- run side by side with the stock binary on the same FASTA files: same command line, the .1aln written
by the reference's own writer, the PAF by the reference's own ALNtoPAF."""
import os
import subprocess
import tempfile

import pytest

import edge_cases
import oracle_lib as ol
from fastga_b200 import formats, synth

pytestmark = pytest.mark.gpu
DROPIN = os.path.join(ol.REF_DIR, "b200", "FastGA")


def _run(binary, args, wd):
    r = subprocess.run([binary] + args, cwd=wd, env=ol.ref_env(), stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout, r.stderr


def _pair(wd, seed, total, ncontig, div, sv):
    A, B = synth.make_pair(seed, total, ncontig, div, sv_every=sv)
    formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", 2))
    formats.write_fasta(os.path.join(wd, "B.fasta"), synth.scaffolds_of(B, "sb", 1))


@pytest.mark.skipif(not (ol.have_ref() and os.path.exists(DROPIN)), reason="oracle/_ref/b200/FastGA not built")
def test_dropin_1aln_equals_stock_binary():
    with tempfile.TemporaryDirectory() as wd:
        _pair(wd, 31, 3_000_000, 4, 0.05, 60_000)
        _same_1aln(wd)


@pytest.mark.skipif(not (ol.have_ref() and os.path.exists(DROPIN)), reason="oracle/_ref/b200/FastGA not built")
def test_dropin_1aln_equals_stock_binary_past_255_contigs():
    """the icont_straddles pair of tests/edge_cases.py: 300 A contigs, so the hook converts records
    whose contig ids do not fit a byte, from seeds whose icont field straddles bit 64"""
    A, B, _, _ = edge_cases.icont_straddles()
    with tempfile.TemporaryDirectory() as wd:
        formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", 1))
        formats.write_fasta(os.path.join(wd, "B.fasta"), synth.scaffolds_of(B, "sb", 1))
        ref = _same_1aln(wd)
        assert max(int(r.split()[1]) for r in ref) > 255


def _same_1aln(wd):
    """stock FastGA and the drop-in on A and B in wd: same canonical records, same -v counters"""
    stock = os.path.join(ol.REF_DIR, "FastGA")
    _, log_ref = _run(stock, ["-v", "-k", "-T8", "-P" + wd, "-1:ref", "A", "B"], wd)
    _, log_b200 = _run(DROPIN, ["-v", "-T8", "-P" + wd, "-1:b200", "A", "B"], wd)
    ref = ol.oneview_records(os.path.join(wd, "ref.1aln"))
    got = ol.oneview_records(os.path.join(wd, "b200.1aln"))
    assert len(ref) > 10 and got == ref
    a, b = ol.parse_fastga_log(log_ref), ol.parse_fastga_log(log_b200)      # the -v lines scripts parse
    assert (a["seeds"], a["hits"], a["alns"], a["kept"]) == (b["seeds"], b["hits"], b["alns"], b["kept"])
    return ref


@pytest.mark.skipif(not (ol.have_ref() and os.path.exists(DROPIN)), reason="oracle/_ref/b200/FastGA not built")
def test_dropin_default_paf_and_self_mode():
    with tempfile.TemporaryDirectory() as wd:
        _pair(wd, 32, 1_500_000, 3, 0.08, 50_000)
        stock = os.path.join(ol.REF_DIR, "FastGA")
        # FASTA sources, default PAF output on stdout: FAtoGDB + (stock: GIXmake) + ALNtoPAF run from PATH
        paf_ref, _ = _run(stock, ["-T4", "-P" + wd, "A.fasta", "B.fasta"], wd)
        for f in os.listdir(wd):
            if not f.endswith(".fasta"):
                os.remove(os.path.join(wd, f))
        paf_b200, _ = _run(DROPIN, ["-T4", "-P" + wd, "A.fasta", "B.fasta"], wd)
        assert paf_ref.count("\n") > 5 and sorted(paf_b200.split("\n")) == sorted(paf_ref.split("\n"))
        # SELF mode (one source); -T1 keeps the reference's own output schedule-independent
        _run(stock, ["-k", "-T1", "-P" + wd, "-1:sref", "A"], wd)
        _run(DROPIN, ["-T1", "-P" + wd, "-1:sb200", "A"], wd)
        assert ol.oneview_records(os.path.join(wd, "sb200.1aln")) == ol.oneview_records(os.path.join(wd, "sref.1aln"))

"""The SELF-mode inputs of self_cases.py without a GPU: every crafted table reaches the corner of the self
merge it is named for, on the oracle; the straddle and divergence genomes reach the main-diagonal branch of
align_contigs, the oracle in the reference's mode gives the records of the reference's `FastGA -T1 A`
(tests/golden/reference_runs.json), the CUDA path's advance differs from it by a stated number of records,
and every bordered Local_Alignment call of the search equals the reference's."""
import os

import numpy as np
import pytest

import oracle_lib as ol
import self_cases as sc
from fastga_b200 import formats, synth


def _seeds(T, freq):
    return ol.self_merge(T.tab, T.pstart(), freq)


@pytest.mark.parametrize("name", sorted(sc.TABLES))
def test_table_reaches_its_regime(name):
    T = sc.table(name)
    pstart = T.pstart()
    pre = (T.tab[:, 1] >> np.uint64(40)).astype(np.int64)
    assert (np.diff(pre) >= 0).all() and pstart[-1] == T.n
    # a block seeds exactly when it has fewer than freq members, every member against every other
    for f in sc.FREQS:
        s, _ = _seeds(T, f)
        yes, no = T.seeding_posts(f)
        ip = set(s["ipost"].tolist())
        assert set(yes.tolist()) <= ip and not (set(no.tolist()) & ip), f
        if f <= 2:
            assert len(s) == 0
    s10, _ = _seeds(T, 10)
    ms = [b.m for b in T.blocks]
    if name == "freq_blocks":
        for f in sc.FREQS:
            assert {f - 1, f, f + 1, 3 * f + 5} - {0, 1} <= set(ms)
        assert {(b.m, b.plen) for b in T.blocks} >= {(m, p) for m in (2, 3, 4) for p in (12, 31, 32, 33, 39, 40)}
    if name == "plen_sweep":
        assert set(s10["plen"].tolist()) >= set(range(12, 41))
    if name == "panels":
        for p in (0, (1 << 24) - 1):
            assert pstart[p + 1] - pstart[p] > 20
        panel_of = {int(v): int(q) for v, q in zip(T.tab[:, 0] & np.uint64(0xffffffff), pre)}
        seeded = {panel_of[int(v)] for v in s10["ipost"]}
        assert {0, (1 << 24) - 1} <= seeded
        assert ((np.diff(pstart) == 1).sum()) > 100                      # singleton panels
    if name == "strands":
        assert set(s10["comp"].tolist()) == {0, 1}
        assert ((s10["ipost"] == s10["jpost"]) & (s10["comp"] == 1)).sum() >= 6   # the palindromes
    if name.startswith("n2"):
        assert T.n == int(name[1:])
    if name == "large":
        assert T.n > 1_000_000
    if name == "overflow":
        assert len(s10) > 2 * T.n + 1024
    if name == "contigs2b":
        assert T.ncontig > 256 and max(s10["icont"].max(), s10["jcont"].max()) > 255


@pytest.mark.parametrize("name", sorted(sc.GENOMES))
def test_self_genome_reaches_the_main_diagonal_branch(name):
    ref = sc.SelfRun(sc.GENOMES[name](), straddle_zero=False)
    zero = sc.SelfRun(sc.GENOMES[name](), straddle_zero=True)
    print(name, "reference mode", ref.counters, "zero mode", zero.counters)
    assert ref.counters["straddles"] > 0
    # with the zero advance (what the device runs): calls on both sides of the main diagonal
    assert zero.counters["lbord_calls"] > 0 and zero.counters["hbord_calls"] > 0
    if name == "divergence":
        assert ref.counters["stale_straddles"] > 0
    rec = lambda R: [tuple(int(r[f]) for f in ol.OVL_DT.names if f != "toff") for r in R.ov]
    got, want = rec(zero), rec(ref)
    if name == "divergence":
        assert set(want) < set(got) and len(got) - len(want) == sc.DIVERGENT_RECORDS
    else:
        assert got == want


@pytest.mark.parametrize("name", sorted(sc.GENOMES))
def test_self_genome_vs_reference_single_thread(name, tmp_path):
    """`FastGA -T1 A` (one thread: the one Path whose stale bepos the straddle reads is the oracle's) against
    the oracle in the reference's mode, and the zero advance DIVERGENT_RECORDS records away from it"""
    G = sc.GENOMES[name]()
    wd = str(tmp_path)
    formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(G, "sa", 1))
    st = ol.reference("self/%s_T1" % name, ol.digest(G), lambda: ol.ref_alignments(wd, "A", None, threads=1))
    g = formats.genome_from_arrays(G)
    r = ol.oracle_pipeline_self(g)
    assert r["nseeds"] // 2 == st["seeds"]
    assert r["nhit"] == st["hits"] and r["nraw"] == st["alns"]
    assert len(r["lines"]) == st["records"] and ol.md5_lines(r["lines"]) == st["aln_md5"]
    ol.check_filters_and_order(r, st)
    z = ol.oracle_pipeline_self(g, straddle_zero=True)
    assert z["nhit"] == r["nhit"]
    extra = sc.DIVERGENT_RECORDS if name == "divergence" else 0
    assert z["nraw"] - r["nraw"] == extra
    assert len(set(z["lines"]) ^ set(r["lines"])) == extra


@pytest.mark.parametrize("name", sorted(sc.GENOMES))
def test_bordered_calls_match_reference_local_alignment(name):
    R = sc.SelfRun(sc.GENOMES[name]())
    want = R.reference_keys(name)
    assert [ol.call_key(c) for c in R.calls] == want
    assert any(c["lbord"] >= 0 for c in R.calls) and any(c["hbord"] >= 0 for c in R.calls)
    if ol.have_ref():
        assert ol.ref_local_alignments(R.call_args(), R.g.freq) == want

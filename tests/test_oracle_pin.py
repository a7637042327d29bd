"""CPU tests that pin the oracle (oracle/fastga_oracle.c) to the UNMODIFIED reference:
  * golden vectors (tests/golden/reference_golden.json, made by tests/golden/make_golden.py);
  * the reference's results on further inputs (libfastga_ref.so Local_Alignment, FastGA runs), stored
    in tests/golden/reference_runs.json by oracle_lib.reference;
  * one check that the reference's own tools read what formats.write_1aln_ascii writes, which needs
    oracle/_ref itself (skipped where it has not been built)."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import oracle_lib as ol
from fastga_b200 import formats, synth

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_golden.json")))


def _pair(c):
    A, B = synth.make_pair(c["seed"], c["total"], c["ncontig"], c["div"], sv_every=c["sv"])
    return formats.genome_from_arrays(A), formats.genome_from_arrays(B)


@pytest.mark.parametrize("name", sorted(GOLD))
def test_oracle_reproduces_reference_golden(name):
    g = GOLD[name]
    gA, gB = _pair(g["case"])
    r = ol.oracle_pipeline(gA, gB)
    cnt = g["counters"]
    assert r["nseeds"] == cnt["seeds"]
    assert abs(r["sumlen"] / r["nseeds"] - cnt["avelen"]) < 0.051
    assert r["nhit"] == cnt["hits"] == r["nchain"]
    assert r["nraw"] == cnt["alns"]
    assert len(r["lines"]) == cnt["kept"] == g["aln_records"]
    assert r["lines"][:3] == g["first_records"]
    assert ol.md5_lines(r["lines"]) == g["aln_md5"]          # bit-exact .1aln content
    for nm, genome, tab, pstart in (("A", gA, r["tabA"], r["pstartA"]), ("B", gB, r["tabB"], r["pstartB"])):
        gg = g["gix"][nm]
        assert hashlib.md5(genome.bps.tobytes()).hexdigest() == gg["bps_md5"]
        assert len(tab) == gg["n"]
        pb, cb = formats.gix_bytes(genome)
        assert (pb, cb) == (gg["post_bytes"], gg["cont_bytes"])
        index = pstart[1:].astype(np.int64)                  # stub index = cumulative counts
        assert hashlib.md5(index.tobytes()).hexdigest() == gg["index_md5"]
        part_first = np.cumsum([0] + gg["part_n"][:-1])
        ent = formats.ktab_entries_from_table(tab, pb, cb, part_first)
        E = 9 + pb + cb                                      # .ktab bytes, equal k-mers canonicalised
        assert hashlib.md5(formats.canonical_ktab(ent, E, index).tobytes()).hexdigest() == gg["entries_md5"]


# ---------------------------------------------------------------------------------------------
#  live pins against oracle/_ref
# ---------------------------------------------------------------------------------------------

class OPath(C.Structure):
    _fields_ = [("abpos", C.c_int), ("bbpos", C.c_int), ("aepos", C.c_int), ("bepos", C.c_int),
                ("diffs", C.c_int), ("tlen", C.c_int), ("trace", C.POINTER(C.c_uint8)), ("tmax", C.c_int)]


def _mutate(rng, a, rate):
    out, i = [], 0
    r = rng.random(len(a) * 2 + 8)
    q = 0
    while i < len(a):
        u = r[q]
        q += 1
        if u < rate * 0.8:
            out.append((a[i] + rng.integers(1, 4)) % 4)
            i += 1
        elif u < rate * 0.9:
            out.append(rng.integers(0, 4))
        elif u < rate:
            i += 1
        else:
            out.append(a[i])
            i += 1
    return np.array(out, dtype=np.int8)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_local_alignment_bit_exact_vs_reference_library(seed):
    _la_compare(seed, borders=False)


@pytest.mark.parametrize("seed", [11, 12])
def test_local_alignment_with_band_borders_vs_reference_library(seed):
    """lbord / hbord >= 0 confine the band to [low-lbord, hgh+hbord] (align.c:1466-1481): what
    align_contigs passes for a contig against itself (FastGA.c:3247-3262); the CUDA waves take the
    same minp/maxp arguments but FastGA's non-self mode never sets them"""
    _la_compare(seed, borders=True)


def _la_calls(seed, borders):
    rng = np.random.default_rng(seed)
    calls = []
    for it in range(400):
        L = int(rng.integers(300, 5000))
        rate = float(rng.choice([0.0, 0.02, 0.05, 0.1, 0.15, 0.3]))
        core = rng.integers(0, 4, L).astype(np.int8)
        fa, fb, ta, tb = (rng.integers(0, 4, int(rng.integers(0, 400))).astype(np.int8) for _ in range(4))
        if rng.random() < 0.3:
            fa = fa[:0]
        if rng.random() < 0.3:
            tb = tb[:0]
        a = np.concatenate([fa, core, ta])
        b = np.concatenate([fb, _mutate(rng, core, rate), tb])
        acomp = int(rng.random() < 0.5)
        xa, xb = len(fa) + L // 2, len(fb) + L // 2
        d, anti = xa - xb, xa + xb + int(rng.integers(-100, 100))
        low, hgh = d - int(rng.integers(0, 80)), d + int(rng.integers(0, 80))
        lb = hb = -1
        if borders:
            lb = int(rng.integers(0, 40)) if rng.random() < 0.7 else -1
            hb = int(rng.integers(0, 40)) if rng.random() < 0.7 else -1
        calls.append((ol._framed(a), ol._framed(b), acomp, low, hgh, anti, lb, hb))
    return calls


def _la_compare(seed, borders, ave_corr=0.7, freq=None):
    """the oracle's Local_Alignment against the reference's on _la_calls(seed, borders); at the default
    spec (ave_corr .7, uniform freq) under the original keys, else under keys that name both"""
    calls = _la_calls(seed, borders)
    name = "local_alignment/%d%s" % (seed, "_borders" if borders else "")
    if freq is None and ave_corr == 0.7:
        freq = np.array([.25] * 4, np.float32)
        want = ol.reference(name, ol.digest(calls), lambda: ol.ref_local_alignments(calls, freq))
    else:
        freq = np.array([.25] * 4, np.float32) if freq is None else np.asarray(freq, np.float32)
        name += "_i%.3g_at%.3g" % (ave_corr, float(freq[0]) + float(freq[3]))
        want = ol.reference(name, ol.digest(calls, ave_corr, freq),
                            lambda: ol.ref_local_alignments(calls, freq, ave_corr))
    _la_check_oracle(calls, want, freq, ave_corr)


def _la_check_oracle(calls, want, freq, ave_corr):
    """every call through the oracle's Local_Alignment gives the reference's path_key want[call]"""
    orc = ol.orc()
    orc.orc_local_alignment.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int] + \
        [C.c_int] * 6 + [C.POINTER(OPath)]
    ospec, _tabs, _ = ol.make_spec(freq, ave_corr)
    owork = C.c_void_p(orc.orc_new_work())
    for it, (ab, bb, acomp, low, hgh, anti, lb, hb) in enumerate(calls):
        op = OPath()
        orc.orc_local_alignment(owork, C.byref(ospec), ab.ctypes.data + 1, len(ab) - 2, bb.ctypes.data + 1,
                                len(bb) - 2, acomp, low, hgh, anti, lb, hb, C.byref(op))
        ot = np.ctypeslib.as_array(op.trace, shape=(max(op.tlen, 1),))[:op.tlen] if op.tlen else np.zeros(0, np.uint8)
        got = ol.path_key(op.abpos, op.bbpos, op.aepos, op.bepos, op.diffs, op.tlen, ot)
        assert got == want[it], (it, acomp, low, hgh, anti, lb, hb,
                                 (op.abpos, op.bbpos, op.aepos, op.bepos, op.diffs, op.tlen))


def test_oracle_vs_live_reference_run(tmp_path):
    A, B = synth.make_pair(31, 600_000, 3, 0.07, sv_every=30_000)
    wd = str(tmp_path)
    formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", 1))
    formats.write_fasta(os.path.join(wd, "B.fasta"), synth.scaffolds_of(B, "sb", 3))

    def run():
        st = ol.ref_alignments(wd, "A", "B", threads=4)
        clen, names, scaf, sbeg = ol.read_gdb_ascii(os.path.join(wd, "B.1gdb"))
        st.update(clen=clen.tolist(), scaf=scaf.tolist(), sbeg=sbeg.tolist())
        return st
    st = ol.reference("oracle/pair31", ol.digest(A, B), run)
    gA = formats.genome_from_fasta(os.path.join(wd, "A.fasta"))
    gB = formats.genome_from_fasta(os.path.join(wd, "B.fasta"))
    assert st["clen"] == gB.clen.tolist() and st["sbeg"] == gB.sbeg.tolist() and st["scaf"] == gB.scaf.tolist()
    r = ol.oracle_pipeline(gA, gB)
    assert (r["nseeds"], r["nhit"], r["nraw"], len(r["lines"])) == (st["seeds"], st["hits"], st["alns"], st["kept"])
    assert len(r["lines"]) == st["records"] and ol.md5_lines(r["lines"]) == st["aln_md5"]
    ol.check_filters_and_order(r, st)


@pytest.mark.skipif(not ol.have_ref(), reason="oracle/_ref not built")
def test_written_1aln_is_read_by_reference_tools(tmp_path):
    """SURVEY 8 a-16: a .1aln written by formats.write_1aln_ascii is accepted by the reference's
    ONEview (same records back) and -- after ONEview -b adds the binary index the threaded readers
    need -- by its ALNtoPAF next to the reference-made GDBs (same PAF as from the reference's own
    .1aln)."""
    A, B = synth.make_pair(41, 500_000, 3, 0.06, sv_every=40_000)
    wd = str(tmp_path)
    formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", 2))
    formats.write_fasta(os.path.join(wd, "B.fasta"), synth.scaffolds_of(B, "sb", 1))
    ol.ref_fastga(wd, "A", "B", threads=4)
    gA = formats.genome_from_fasta(os.path.join(wd, "A.fasta"))
    gB = formats.genome_from_fasta(os.path.join(wd, "B.fasta"))
    r = ol.oracle_pipeline(gA, gB)
    formats.write_1aln_ascii(os.path.join(wd, "mine.1aln"), r["alns"], gA, gB, "./A.1gdb", "./B.1gdb", wd)
    assert ol.oneview_records(os.path.join(wd, "mine.1aln")) == ol.oneview_records(os.path.join(wd, "ref.1aln"))
    paf_ref = sorted(ol.run_ref(["ALNtoPAF", "-T2", "ref"], cwd=wd).split("\n"))
    # the threaded converters need ONEcode's binary index: ONEview -b turns the ASCII file into it
    ol.run_ref(["ONEview", "-b", "-o", "mineb.1aln", "mine.1aln"], cwd=wd)
    paf_mine = sorted(ol.run_ref(["ALNtoPAF", "-T2", "mineb"], cwd=wd).split("\n"))
    assert len(paf_ref) > 3 and paf_mine == paf_ref


import edge_cases  # noqa: E402


@pytest.mark.parametrize("name", sorted(edge_cases.CASES))
def test_oracle_edge_cases_vs_live_reference(name):
    """the oracle on the edge-case inputs of tests/edge_cases.py, against the reference's run"""
    A, B, threads, check = edge_cases.CASES[name]()
    st = edge_cases.reference_run(name)
    r = ol.oracle_pipeline(formats.genome_from_arrays(A), formats.genome_from_arrays(B))
    assert r["nseeds"] == st.get("seeds", 0)
    assert r["nhit"] == st.get("hits", 0) == r["nchain"] and r["nraw"] == st.get("alns", 0)
    assert len(r["lines"]) == st["records"] and ol.md5_lines(r["lines"]) == st["aln_md5"]
    ol.check_filters_and_order(r, st)
    check(r["alns"], r["nhit"])


def test_max_contigs_records_do_not_depend_on_the_filler_tie_order():
    """the max_contigs fillers have repeated lengths, so their ranks depend on how a sort breaks ties
    (the reference's and the library's libc qsort, the oracle's stable argsort).  Ties broken the other
    way round give the reference's records too, which is what lets the case be compared at all."""
    A, B, _, _ = edge_cases.max_contigs()
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    st = edge_cases.reference_run("max_contigs")
    perm = np.lexsort((-np.arange(gA.ncontig), -gA.clen))          # equal lengths: last index first
    ra = np.empty(gA.ncontig, np.int32)
    ra[perm] = np.arange(gA.ncontig)
    assert not np.array_equal(ra, ol.contig_rank(gA.clen)[1])
    r = ol.oracle_pipeline(gA, gB, rank=(ra, ol.contig_rank(gB.clen)[1]))
    assert r["nseeds"] == st["seeds"]
    assert len(r["lines"]) == st["records"] and ol.md5_lines(r["lines"]) == st["aln_md5"]
    ol.check_filters_and_order(r, st)


def test_oracle_on_example_regions_vs_live_reference(tmp_path):
    """the EXAMPLE regions fixture of the GPU regression test, oracle against the reference's run"""
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "example_regions.npz"))
    A = [z["a%d" % i] for i in range(10)]
    B = [z["b%d" % i] for i in range(10)]
    wd = str(tmp_path)
    formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", 1))
    formats.write_fasta(os.path.join(wd, "B.fasta"), synth.scaffolds_of(B, "sb", 1))
    st = ol.reference("oracle/example_regions", ol.digest(A, B), lambda: ol.ref_alignments(wd, "A", "B", threads=4))
    r = ol.oracle_pipeline(formats.genome_from_arrays(A), formats.genome_from_arrays(B))
    assert r["nseeds"] == st.get("seeds", 0)
    assert len(r["lines"]) == st["records"] and ol.md5_lines(r["lines"]) == st["aln_md5"]
    ol.check_filters_and_order(r, st)


def _self_genomes():
    """genomes with internal homology for SELF mode (FastGA A): a diverged duplication inside and
    across contigs plus an inverted copy, and two tandem-repeat genomes (near-diagonal chains: the band
    borders of align_contigs).  None of them reaches the 'nothing across the main diagonal' branch:
    self_cases.py builds the genomes that do."""
    rng = np.random.default_rng(5)
    a = rng.integers(0, 4, 300_000, dtype=np.uint8)
    dup = synth.diverged_copy(rng, a[50_000:150_000], 0.05, sv_every=40_000)
    c0 = np.concatenate([a, dup, rng.integers(0, 4, 20_000, dtype=np.uint8)])
    c1 = np.concatenate([rng.integers(0, 4, 100_000, dtype=np.uint8),
                         synth.diverged_copy(rng, a[200_000:280_000], 0.04, sv_every=30_000),
                         (3 - a[10_000:60_000][::-1]).astype(np.uint8)])
    out = {"dup": [c0, c1[:len(c1) - 3]]}
    for seed in (61, 62):
        rng = np.random.default_rng(seed)
        parts = []
        while sum(len(p) for p in parts) < 500_000:
            parts.append(rng.integers(0, 4, int(rng.integers(20_000, 60_000)), dtype=np.uint8))
            unit = rng.integers(0, 4, int(rng.integers(150, 1200)), dtype=np.uint8)
            parts.append(np.concatenate([synth._small_mutations(rng, unit, 0.03)
                                         for _ in range(int(rng.integers(8, 60)))]))
        g = np.concatenate(parts)[:500_000]
        cut = int(rng.integers(200_000, 300_000))
        out["tandem%d" % seed] = [g[:cut], g[cut:]]
    # C-strand self pairs, identical contigs, a palindrome, a long near-diagonal repeat array
    rng = np.random.default_rng(101)
    a = rng.integers(0, 4, 200_000, dtype=np.uint8)
    inv = (3 - a[30_000:90_000][::-1]).astype(np.uint8)
    out["inverted_dup"] = [np.concatenate([a, rng.integers(0, 4, 5000, dtype=np.uint8),
                                           synth._small_mutations(rng, inv, 0.03)])]
    out["identical_contigs"] = [a.copy(), a.copy()[:199_990], rng.integers(0, 4, 50_000, dtype=np.uint8)]
    out["palindrome"] = [np.concatenate([a[:60_000], (3 - a[:60_000][::-1]).astype(np.uint8)]),
                         rng.integers(0, 4, 30_001, dtype=np.uint8)]
    rng = np.random.default_rng(102)
    unit = rng.integers(0, 4, 5000, dtype=np.uint8)
    out["near_diagonal_repeats"] = [np.concatenate(
        [rng.integers(0, 4, 50_000, dtype=np.uint8)] +
        [synth._small_mutations(rng, unit, 0.04) for _ in range(30)] +
        [rng.integers(0, 4, 50_000, dtype=np.uint8)])]
    # 300 contigs with a 600 kbp longest: a 67-bit seed key whose icont field straddles bit 64;
    # every other short contig is a diverged copy of a piece of the long one
    rng = np.random.default_rng(103)
    a = rng.integers(0, 4, 600_000, dtype=np.uint8)
    g = [np.concatenate([a[:540_000], synth.diverged_copy(rng, a[100_000:160_000], 0.05, sv_every=0)])]
    for k in range(299):
        n = int(rng.integers(2_000, 6_000))
        s = int(rng.integers(0, 600_000 - n))
        g.append(synth._small_mutations(rng, a[s:s + n], 0.05) if k % 2 else rng.integers(0, 4, n, dtype=np.uint8))
    out["contigs300"] = edge_cases._distinct(g)
    return out


@pytest.mark.parametrize("name", ["dup", "tandem61", "tandem62", "inverted_dup", "identical_contigs",
                                  "palindrome", "near_diagonal_repeats", "contigs300"])
def test_oracle_self_mode_vs_live_reference(name, tmp_path):
    """SURVEY row a-7 groundwork: the oracle's SELF mode (self block rule, band borders for a contig
    against itself) against `FastGA A` of the reference"""
    G = _self_genomes()[name]
    wd = str(tmp_path)
    formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(G, "sa", 1))
    st = ol.reference("self/" + name, ol.digest(G), lambda: ol.ref_alignments(wd, "A", None, threads=4))
    r = ol.oracle_pipeline_self(formats.genome_from_arrays(G))
    # every thread of the reference halves its own pair count (FastGA.c:1907): off by < #threads
    assert abs(r["nseeds"] // 2 - st["seeds"]) < 4
    assert r["nhit"] == st["hits"] and r["nraw"] == st["alns"]
    assert len(r["lines"]) == st["records"] and ol.md5_lines(r["lines"]) == st["aln_md5"]
    ol.check_filters_and_order(r, st)

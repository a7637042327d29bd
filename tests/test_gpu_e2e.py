"""-m gpu: the reference-facing call (fgb_fastga, host buffers) against the UNMODIFIED reference
(oracle/_ref/FastGA; its results stored in tests/golden/reference_runs.json), records compared
bit-exactly after the canonical sort."""
import hashlib
import os
import tempfile

import numpy as np
import pytest

import oracle_lib as ol
from fastga_b200 import formats, lib, synth

pytestmark = pytest.mark.gpu


def _vs_reference(name, seed, total, ncontig, div, sv, threads=8, per_scaffold=1):
    A, B = synth.make_pair(seed, total, ncontig, div, sv_every=sv)
    with tempfile.TemporaryDirectory() as wd:
        formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", per_scaffold))
        formats.write_fasta(os.path.join(wd, "B.fasta"), synth.scaffolds_of(B, "sb", per_scaffold))
        gA = formats.genome_from_fasta(os.path.join(wd, "A.fasta"))
        gB = formats.genome_from_fasta(os.path.join(wd, "B.fasta"))

        def run():
            st = ol.ref_alignments(wd, "A", "B", threads)
            st["bps_md5"] = hashlib.md5(open(os.path.join(wd, ".A.bps"), "rb").read()).hexdigest()
            return st
        st = ol.reference("e2e/" + name, ol.digest(A, B, threads, per_scaffold), run)
    assert hashlib.md5(gA.bps.tobytes()).hexdigest() == st["bps_md5"]
    alns, stats = lib.fastga(gA, gB)
    assert stats["nseeds"] == st["seeds"]
    assert stats["nhits"] == st["hits"]
    assert alns.nraw == st["alns"]
    assert len(alns) == st["kept"] == st["records"]
    assert ol.md5_lines(alns.canonical_lines()) == st["aln_md5"]
    return stats


def test_small_pair_bit_exact_vs_reference():
    _vs_reference("small_pair", 11, 1_200_000, 3, 0.05, 60_000)


def test_scaffolded_15pct_bit_exact_vs_reference():
    _vs_reference("scaffolded_15pct", 12, 2_000_000, 6, 0.15, 40_000, per_scaffold=3)


def test_long_alignments_exercise_arena_retry():
    # no SV breaks: contig-long alignments -> pebble arenas overflow and the retry path runs
    _vs_reference("long_alignments", 13, 6_000_000, 3, 0.03, 0)


def test_10mbp_bit_exact_vs_reference():
    _vs_reference("10mbp", 14, 10_000_000, 5, 0.05, 200_000)


@pytest.mark.parametrize("gap", ["0", "3000", "1000000000"])
def test_hit_groups_any_cut_gives_the_same_records(gap):
    # The extension runs the hits of a band-pair triple as independent groups and re-runs the triple in
    # one piece when a group's alignments reached into the next group (fgb_extend).  Cutting at every
    # hit (0: covered hits are aligned speculatively, found out, re-run), at 3 kbp, or never must all
    # give the records of the default cut.
    A, B = synth.make_pair(21, 3_000_000, 4, 0.08, sv_every=50_000)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    base, st0 = lib.fastga(gA, gB)
    os.environ["FGB_SPEC_GAP"] = gap
    try:
        alns, st1 = lib.fastga(gA, gB)
    finally:
        del os.environ["FGB_SPEC_GAP"]
    assert st1["nhits"] == st0["nhits"] and alns.nraw == base.nraw
    assert ol.md5_lines(alns.canonical_lines()) == ol.md5_lines(base.canonical_lines())


def test_smoke_entry():
    import __graft_entry__
    __graft_entry__.smoke()


def test_example_regions_wide_band_chunks_bit_exact_vs_oracle():
    """ten 25-40 kbp regions of EXAMPLE (tests/golden/example_regions.npz) whose alignments run
    through bands wider than one 32-lane chunk with the fresh low edge alone in the last chunk: the
    case where the edge must copy the OLD trace-point counter of the diagonal that closed the
    previous chunk (a missing trace point otherwise; found on the full EXAMPLE)"""
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "example_regions.npz"))
    gA = formats.genome_from_arrays([z["a%d" % i] for i in range(10)])
    gB = formats.genome_from_arrays([z["b%d" % i] for i in range(10)])
    want = ol.oracle_pipeline(gA, gB)
    alns, stats = lib.fastga(gA, gB)
    assert stats["nseeds"] == want["nseeds"] and stats["nhits"] == want["nhit"]
    assert alns.canonical_lines() == want["lines"]


def _gixmake_genome(name):
    """(contigs, contigs per scaffold): pair17, and genomes on either side of the .ktab field widths --
    cont_bytes 1 -> 2 between 128 and 129 contigs, post_bytes 3 -> 4 between a longest contig of
    2^24 and 2^24 + 1"""
    if name == "pair17":
        return synth.make_pair(17, 2_500_000, 5, 0.05, sv_every=100_000)[0], 2
    rng = np.random.default_rng(18)
    if name.startswith("contigs"):
        n = int(name[len("contigs"):])
        return [rng.integers(0, 4, int(k), dtype=np.uint8) for k in rng.choice(np.arange(2_000, 6_000), n, replace=False)], 1
    maxlen = {"maxlen_2_24": 1 << 24, "maxlen_2_24_plus_1": (1 << 24) + 1}[name]
    return [rng.integers(0, 4, 200_000, dtype=np.uint8), rng.integers(0, 4, maxlen, dtype=np.uint8),
            rng.integers(0, 4, 90_001, dtype=np.uint8)], 1


GIXMAKE_GENOMES = {"pair17": (3, 1), "contigs128": (2, 1), "contigs129": (2, 2),
                   "maxlen_2_24": (3, 1), "maxlen_2_24_plus_1": (4, 1)}      # (post_bytes, cont_bytes)


def gixmake_reference(name):
    """what the reference GIXmake writes for _gixmake_genome(name)"""
    A, per_scaffold = _gixmake_genome(name)

    def run():
        with tempfile.TemporaryDirectory() as wd:
            formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", per_scaffold))
            ol.run_ref(["GIXmake", "-T4", "-P" + wd, "A"], cwd=wd)
            ref = formats.read_gix(os.path.join(wd, "A.gix"))
        return {"n": int(ref.n), "post_bytes": ref.post_bytes, "cont_bytes": ref.cont_bytes, "esize": ref.esize,
                "index_md5": hashlib.md5(ref.index.astype(np.int64).tobytes()).hexdigest(),
                "perm": [int(x) for x in ref.perm], "nparts": ref.nparts, "ncontig": ref.ncontig, "part_n": [int(x) for x in ref.part_n],
                "entries_md5": hashlib.md5(formats.canonical_ktab(ref.entries, ref.esize, ref.index).tobytes()).hexdigest()}
    return A, ol.reference("gixmake/" + name, ol.digest(A), run)


def test_gix_files_match_reference_gixmake():
    """SURVEY 8 a-4: the .ktab entry stream, the stub index, the part split and the contig order
    produced from the device table equal what the reference GIXmake writes (equal k-mers
    canonicalised), and that entry stream imports back into the identical device table"""
    _gixmake_compare("pair17")


@pytest.mark.parametrize("name", ["contigs128", "contigs129", "maxlen_2_24", "maxlen_2_24_plus_1"])
def test_gix_files_match_reference_gixmake_at_field_widths(name):
    """the same comparison on either side of the .ktab contig and post field widths"""
    _gixmake_compare(name)


def _gixmake_compare(name):
    A, ref = gixmake_reference(name)
    assert (ref["post_bytes"], ref["cont_bytes"]) == GIXMAKE_GENOMES[name]
    g = formats.genome_from_arrays(A)
    dg = lib.DeviceGenome(g)
    gx = lib.DeviceGix.build(dg)
    tab, pstart, buck = gx.download()
    assert gx.n == ref["n"]
    pb, cb = formats.gix_bytes(g)
    assert (pb, cb) == (ref["post_bytes"], ref["cont_bytes"]) == (gx.post_bytes, max(gx.cont_bytes, cb))
    index = pstart[1:].astype(np.int64)
    assert hashlib.md5(index.tobytes()).hexdigest() == ref["index_md5"]
    assert list(dg.perm) == ref["perm"][:g.ncontig]
    # part split from the sampler histogram (GIXmake.c:655-691)
    nparts = formats.gix_nparts(g.seqtot, max(g.ncontig, 4), pb, cb, nthreads=4)
    assert nparts == ref["nparts"]
    ks = formats.ksplit_from_buckets(buck, nparts)
    part_first = np.array([int(pstart[k << 14]) for k in ks[:-1]], dtype=np.int64)
    part_n = np.diff(np.concatenate([part_first, [gx.n]]))
    assert list(part_n) == ref["part_n"]
    ent = gx.export_ktab(part_first) if gx.cont_bytes == cb else None
    if ent is None:     # device handle counts real contigs only; re-encode with the padded width
        ent = formats.ktab_entries_from_table(tab, pb, cb, part_first)
    E = ref["esize"]
    assert hashlib.md5(formats.canonical_ktab(ent, E, index).tobytes()).hexdigest() == ref["entries_md5"]
    # and the reverse direction: .ktab entries (the reference's, up to the order of equal k-mers) -> device table
    gf = formats.GixFile()
    gf.entries, gf.n, gf.post_bytes, gf.cont_bytes, gf.index, gf.ncontig = ent, gx.n, pb, cb, index, ref["ncontig"]
    imp = lib.DeviceGix.import_ktab(gf)
    itab, ipstart, _ = imp.download()
    assert np.array_equal(ipstart, pstart)
    # A reverse-strand post counts from the contig's end, 1 .. length, so a longest contig of exactly
    # 2^24 has one post of 2^24, which the reference's PostBytes rule (cum < maxlen, 3 bytes) leaves
    # one byte short: GIXmake writes it truncated (the entries md5 above), and so it comes back.
    post = tab[:, 0] & np.uint64(0xffffffff)
    short = post >> np.uint64(8 * pb) != 0 if pb < 4 else np.zeros(len(tab), bool)
    assert int(short.sum()) == (1 if name == "maxlen_2_24" else 0)
    want = tab.copy()
    want[short, 0] -= post[short] - (post[short] & np.uint64((1 << (8 * pb)) - 1))
    key = lambda t: np.lexsort((t[:, 0] & np.uint64(0xffffffffffff), t[:, 0] >> np.uint64(48), t[:, 1]))
    assert np.array_equal(itab[key(itab)], want[key(want)])


# ---------------------------------------------------------------------------------------------
#  edge cases (tests/edge_cases.py): ragged / degenerate inputs, against the reference
# ---------------------------------------------------------------------------------------------

import edge_cases  # noqa: E402


@pytest.mark.parametrize("name", sorted(edge_cases.CASES))
def test_edge_case_bit_exact_vs_reference(name):
    A, B, threads, check = edge_cases.CASES[name]()
    st = edge_cases.reference_run(name)
    alns, stats = lib.fastga(formats.genome_from_arrays(A), formats.genome_from_arrays(B))
    assert stats["nseeds"] == st.get("seeds", 0)
    assert stats["nhits"] == st.get("hits", 0)
    assert alns.nraw == st.get("alns", 0)
    assert len(alns) == st["records"] and ol.md5_lines(alns.canonical_lines()) == st["aln_md5"]
    check(alns, stats["nhits"])

"""The crafted seed records of seed_stage_cases.py without a GPU: each case hits the edges its builder
claims (checked on the numpy restatement of its triples and on the oracle's chain scan), its records are
the sorted, distinct records of SEED_DT rows, and the cases that carry genomes keep every seed inside its
contig pair.  If a builder drifts, its edge fails here."""
import numpy as np
import pytest

import oracle_lib as ol
import seed_stage_cases as sc


@pytest.mark.parametrize("name", sc.NAMES)
def test_case_hits_its_edges(name):
    C = sc.case(name)
    assert C.edges, name
    F = C.facts
    for what, pred in C.edges:
        assert pred(F), "%s: %s" % (name, what)
    # sorted, distinct above the lcp field (so a sort from bit 6 gives the same order), keys of <= 64 bits
    lo = C.recs[:, 0]
    assert not C.recs[:, 1].any()
    assert (np.diff(lo >> np.uint64(6)) > 0).all()
    assert 12 + sum(C.layout[:4]) + 1 <= 64
    if C.genomes is not None:
        assert C.posts_ok, name
    # the oracle's triples are the numpy restatement's scanned ones, with the same extents
    assert np.array_equal(F.otr["b"], F.seg[F.scanned]) and np.array_equal(F.otr["e"], F.e[F.scanned])
    assert bool((F.otr["isnew"] != 0).tolist() == F.isnew[F.scanned].tolist())
    # what the prefilter drops holds no chain
    assert all(F.nh[int(b)] == 0 for b in F.seg[F.scanned & ~F.kept])
    assert F.nlong <= F.lcap


def test_seed_rows_pack_to_the_fields_asked_for():
    """seed_rows and seed_records agree on every field, on both strands, bands 0 to the top"""
    rng = np.random.default_rng(3)
    k = 5000
    comp = rng.integers(0, 2, k)
    band = np.where(comp == 0, rng.integers(0, 1 << sc.LAYOUT[1], k), rng.integers(sc.MID - 3000, sc.MID + 3000, k))
    anti = rng.integers(sc.A0, sc.A0 + 100_000, k)
    ic, jc, plen, dlow = rng.integers(0, 4, k), rng.integers(0, 4, k), rng.integers(12, 41, k), rng.integers(0, 64, k)
    rows = sc.seed_rows(sc.LAYOUT, comp, ic, jc, band, anti, plen, dlow)
    d = sc.decode(ol.seed_records(rows, sc.LAYOUT, sort=False), sc.LAYOUT)
    for f, v in (("comp", comp), ("ic", ic), ("jc", jc), ("band", band), ("anti", anti), ("lcp", plen)):
        assert np.array_equal(d[f], v), f


def test_families_cover_the_stage():
    """the tile sizes, tile offsets, prefilter bounds and triple sizes the cases reach together"""
    fam = {sc.case(n).family for n in sc.NAMES}
    assert fam == {"tiles", "adjacency", "prefilter", "short_scan", "long_order", "densest", "past_2^20"}
    ns = {sc.case(n).facts.n for n in sc.NAMES if n.startswith("tiles_") and n not in sc.BIG}
    assert {1, 2, 2047, 2048, 2049, 4095, 4096, 4097} <= ns
    assert any(n % sc.SEG_TILE == 1 and n > 4097 for n in ns) and any(n % sc.SEG_TILE == 2047 and n > 4097 for n in ns)
    assert sc.case("empty").facts.n == 0
    bounds = {(sc.case("prefilter_cm%d" % cm).chain_min, (cm + 79) // 80) for cm in sc.PREFILTER_CMS}
    assert bounds == {(1, 1), (80, 1), (81, 2), (170, 3), (2000, 25)}
    # the short-triple scan: the oracle finds a chain in some marked triples and none in others
    marks = sc.case("short_scan").marks
    assert {h for _, _, h in marks} == {True, False} and len(marks) >= 13

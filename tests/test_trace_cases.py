"""CPU: the crafted trace-point records of tests/trace_cases.py reach their regimes, and -- where
oracle/_ref is built -- the reference's Compute_Trace_PTS agrees with the independent checks there
(replay, per-tile DP, the rule for bad records) and with its stored results, so that both can judge
the device (tests/test_gpu_trace_tiles.py)."""
import numpy as np
import pytest

import oracle_lib as ol
import trace_cases as tc

NAMES = sorted(tc.CASES)


def _slab_bytes(m, n, dcap):
    """trace.cu tile_slab_bytes restated: int16 rows D = -2 .. dcap and int8 rows 0 .. dcap of
    |m - n| + 2 (dcap / 2 + 1) + 4 diagonals, rounded up to 16 bytes"""
    w = abs(m - n) + 2 * (dcap // 2 + 1) + 4
    return ((dcap + 3) * w * 2 + (dcap + 1) * w + 15) & ~15


def first_launch_slab(c):
    """bytes of the slabs the first launch takes: every tile sized from its own diff byte"""
    tot = 0
    for k in range(len(c.fields)):
        for a0, m, b0, n, d in tc.tiles(c.fields[k], c.trace(k)):
            tot += _slab_bytes(m, n, max(d - abs(m - n), 0))
    return tot


def test_tile_edit_distance_small():
    """the row DP against the textbook recurrence on random short pairs"""
    rng = np.random.default_rng(1)
    for _ in range(200):
        a = rng.integers(0, 3, int(rng.integers(0, 12)))
        b = rng.integers(0, 3, int(rng.integers(0, 12)))
        ed, ways = tc.count_optimal_scripts(a, b)
        assert tc.tile_edit_distance(a, b) == ed and ways >= 1
    assert tc.count_optimal_scripts([0, 0], [0]) == (1, 2)
    assert tc.count_optimal_scripts([0, 1], [1, 0]) == (2, 3)


def test_replay_reads_entries_like_alntopaf():
    """B extra base before A position 3 (1-based), then A extra base before B position 7"""
    a = np.array([0, 1, 2, 3, 0, 1, 2, 3], np.uint8)
    b = np.array([0, 1, 3, 2, 3, 0, 2, 3], np.uint8)     # B = A[:2] + 3 + A[2:5] + A[6:]
    f = [0, 0, 0, 0, 0, 8, 8, 2, 2]
    cost, pa, pb = tc.replay([-3, 7], f, a, b)
    assert cost == 2 and list(zip(pa, pb))[2:4] == [(2, 2), (2, 3)]
    assert tc.replay([3, -7], f, a, b)[0] == 4              # signs swapped: another walk, another cost
    with pytest.raises(AssertionError):
        tc.replay([-3, 7, 7], f, a, b)                        # an entry behind the walk


@pytest.mark.parametrize("name", NAMES)
def test_case_reaches_its_regime(name):
    c, want = tc.case(name), tc.REGIMES[name]
    F = c.fields
    bad = tc.expect_bad(c)
    if want.get("strands"):
        assert set(F[:, 0]) == {0, 1}
    if want.get("good"):
        assert (~bad).any()
    if want.get("bad"):
        assert bad.any()
    if "max_diff_over" in want:
        assert max(int(c.trace(k)[0::2].max()) for k in range(len(F)) if F[k, 8]) > want["max_diff_over"]
    if want.get("shapes"):
        seen = set()
        for k in range(len(F)):
            ab, ae, tl = int(F[k, 3]), int(F[k, 5]), int(F[k, 8])
            tl_ = tc.tiles(F[k], c.trace(k))
            seen |= {s for s, hit in (("start_on", ab % 100 == 0), ("start_99", ab % 100 == 99),
                                      ("end_on", ae % 100 == 0), ("end_past1", ae % 100 == 1),
                                      ("tlen2", tl == 2), ("one_base", ae - ab == 1)) if hit}
            for a0, m, b0, n, d in tl_:
                seen |= {s for s, hit in (("badv0", n == 0), ("badv255", n == 255), ("del_ge100", m - n >= 100),
                                          ("ins_ge100", n - m >= 100)) if hit}
        assert set(want["shapes"]) <= seen, set(want["shapes"]) - seen
    if want.get("ends"):
        for comp in (0, 1):
            assert any(F[k, 0] == comp and F[k, 3] == 0 and F[k, 4] == 0 and F[k, 5] == len(c.aseq(k))
                       and F[k, 6] == len(c.bseq(k)) for k in range(len(F)))
    if want.get("short_contig"):
        assert any(len(c.aseq(k)) < 100 and len(c.bseq(k)) < 100 for k in range(len(F)))
    if want.get("hundred_contig"):
        assert any(len(c.aseq(k)) % 100 == 0 and F[k, 5] == len(c.aseq(k)) for k in range(len(F)))
    if want.get("ties"):
        found = False
        for k in range(len(F)):
            a, b = c.aseq(k), c.bseq(k)
            for a0, m, b0, n, d in tc.tiles(F[k], c.trace(k)):
                if tc.count_optimal_scripts(a[a0:a0 + m], b[b0:b0 + n])[1] > 1:
                    found = True
                    break
            if found:
                break
        assert found
    if want.get("understated"):
        eds = tc.tile_eds(c)
        assert any(not bad[k] and F[k, 8] >= 2 and (c.trace(k)[0::2] < np.array(eds[k])).any()
                   for k in range(len(F)))
    if want.get("tlen0"):
        z = F[:, 8] == 0
        assert bad[z].any() and (~bad[z]).any()
    if want.get("slack255"):
        assert any(F[k, 8] and (c.trace(k)[0::2] == 255).all() for k in range(len(F)))
    if "slab_over" in want:
        assert first_launch_slab(c) > want["slab_over"]


@pytest.mark.skipif(not ol.have_ref(), reason="needs oracle/_ref (the reference built from its sources)")
@pytest.mark.parametrize("name", NAMES)
def test_reference_passes_the_independent_checks(name):
    """the reference's scripts replay to their diffs, are optimal tile by tile, and it rejects exactly
    the records the rule rejects; its keys are the stored ones"""
    c = tc.case(name)
    gA, gB = c.genomes()
    got = ol.ref_trace_pts_raw(c.alns(), gA, gB)
    bad = tc.expect_bad(c)
    eds = tc.tile_eds(c)
    assert [r is None for r in got] == list(bad)
    for k, r in enumerate(got):
        if r is not None:
            tc.check_script(r[0], r[1], c.fields[k], c.trace(k), c.aseq(k), c.bseq(k), eds[k])
    assert [("fail" if r is None else ol.script_key(*r)) for r in got] == tc.reference_run(name)

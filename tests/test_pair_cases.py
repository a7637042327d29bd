"""The crafted table pairs of pair_cases.py without a GPU: on every case, at every f it is built for, the
oracle's state-machine merge (orc_merge) equals the declarative restatement of SURVEY A.3, and the
unmodified reference's `FastGA -v` on the same tables written as .gix reports the same seed count and
average length (tests/golden/reference_runs.json); every case reaches the corners of the kernel it is named
for, and together they reach every one of them."""
import numpy as np
import pytest

import oracle_lib as ol
import pair_cases as pc

NAMES = sorted(pc.CASES)

#  what each case is named for: the rows of pair_cases.ROWS it must reach (at one of its f at least)
REACH = {
    "freq_edges": {"ins_start", "byte_loop_f10", "byte_loop_f11", "no_loop_f9", "staged", "desc_out"},
    "runs": {"run7", "run8", "run9", "run16", "run17", "byte_loop_f10", "byte_loop_f11", "no_loop_f9",
             "ins_start", "ins_middle", "ins_end", "plen_tie"},
    "plen_sweep": {"plen_hi", "plen_lo", "plen_base39", "plen40", "plen_tie", "ins_middle"},
    "state_machine": {"ins_start", "ins_middle", "ins_end"},
    "panels": {"prefix0", "prefix_top", "sp_staged", "sp_top_panel", "nbr_other_panel", "tile512"},
    "packed_ceiling": {"packed_ceiling", "two_rounds", "entry_out", "overflow", "tile512"},
    "staging": {"slice_0", "slice_1", "slice_1152", "slice_1153", "words_512", "words_513", "sp_staged", "sp_l1",
                "sp_top_panel", "total_1536", "total_1537", "desc_out", "entry_out", "direct", "tile64",
                "table_start", "slice_end"},
    "strands": {"staged"},
    "forward_only": {"table_end"},
    "widths": {"staged"},
    "overflow": {"overflow"},
    "tiles_1000_2100": {"tile512"}, "tiles_1000_2101": {"tile256"},
    "tiles_1000_4200": {"tile256"}, "tiles_1000_4201": {"tile128"},
    "tiles_1000_8400": {"tile128"}, "tiles_1000_8401": {"tile64"},
    "tiles_1025_1500": {"tile512", "two_rounds"}, "tiles_1535_2000": {"tile512", "two_rounds"},
    "tiles_513_2000": {"tile256"}, "tiles_767_2500": {"tile256"}, "tiles_257_3000": {"tile64"},
    "tiles_383_3000": {"tile128"}, "tiles_129_2000": {"tile64"}, "tiles_191_2000": {"tile64"},
    "tiles_round1": {"round1_only", "two_rounds", "tile512"},
}

#  the branches of orc_merge's walk (oracle/fastga_oracle.c MB_*)
BRANCHES = ("panel", "nlcp_gt", "nlcp_eq_eorun", "nlcp_eq", "nlcp_lt", "rend_skip", "nlcp_lt_eorun", "ext_lb",
            "ext_gt", "ext_full")


def _reached(c):
    out = set()
    for f in c.freqs:
        out |= pc.regimes_of(c, f)[2]
    return out


@pytest.mark.parametrize("name", NAMES)
def test_oracle_merge_equals_the_declarative_rule(name):
    c = pc.case(name)
    ps = c.pstart2()
    for f in c.freqs:
        got, gl = ol.merge(c.T1, c.T2, ps, f)
        want, wl = pc.declarative_merge(c.T1, c.T2, ps, f)
        assert (len(got), gl) == (len(want), wl), f
        L = c.layout()
        assert np.array_equal(ol.seed_records(got, L), ol.seed_records(want, L)), f
        # the kernel's geometry restated: its CTA totals add up to the same count
        assert sum(x["total"] for x in pc.regimes(c.T1, c.T2, ps, f)[0]) == len(want), f


@pytest.mark.parametrize("name", NAMES)
def test_case_reaches_its_regime(name):
    c = pc.case(name)
    missing = REACH.get(name, set()) - _reached(c)
    assert not missing, missing
    if name == "packed_ceiling":
        ctas = pc.regimes_of(c, 255)[0]
        assert len(ctas) == 1 and ctas[0]["rounds"] == [65024, 65024] and ctas[0]["total"] == 130048
    if name == "no_forward":
        assert len(c.T1) > 0 and c.n1 == 0
    if name == "forward_only":
        assert ((c.T1[:, 0] >> np.uint64(47)) & np.uint64(1) == 0).all()
    if name == "strands":
        s, _ = ol.merge(c.T1, c.T2, c.pstart2(), 10)
        assert set(s["comp"].tolist()) == {0, 1}
        # the palindromes: one T2 post seeded on both strands by the same T1 entry
        pairs = {(int(a), int(b), int(k)) for a, b, k in zip(s["ipost"], s["jpost"], s["comp"])}
        assert any((a, b, 1 - k) in pairs for a, b, k in pairs)
        rev = (c.T1[:, 0] >> np.uint64(47)) & np.uint64(1)
        assert rev.any() and (rev == 0).any()
    if name == "widths":
        assert len(c.clen1) > 256 and len(c.clen2) > 256
        assert c.upload_bytes(1) == (4, 2) and c.upload_bytes(2) == (4, 2)
        assert c.key_bits() > 64
        s, _ = ol.merge(c.T1, c.T2, c.pstart2(), 10)
        assert s["ipost"].max() >= 1 << 24 and s["jpost"].max() >= 1 << 24
        assert s["icont"].max() > 255 and s["jcont"].max() > 255
    if name == "overflow":
        s, _ = ol.merge(c.T1, c.T2, c.pstart2(), 10)
        assert len(s) > pc.first_reservation(c.n1)


def test_every_row_of_the_kernel_is_reached():
    reached = set()
    for name in NAMES:
        reached |= _reached(pc.case(name))
    print("rows reached:", sorted(r for r in reached if r in pc.ROWS))
    assert [r for r in pc.ROWS if r not in reached] == []


def test_state_machine_takes_every_branch_of_the_walk():
    """the branches of orc_merge's walk on the dense panels, reverse T1 entries between forward ones"""
    c = pc.case("state_machine")
    ol.merge(c.T1, c.T2, c.pstart2(), 10)
    cnt = np.zeros(len(BRANCHES), dtype=np.int64)
    ol.orc().orc_merge_counters(cnt.ctypes.data_as(ol.C.c_void_p))
    counts = dict(zip(BRANCHES, cnt.tolist()))
    print(counts)
    assert all(v > 0 for v in counts.values()), counts


@pytest.mark.parametrize("name", NAMES)
def test_oracle_merge_matches_the_reference(name):
    """`FastGA -v -f<f>` on the case's tables (pair_cases.ref_merge): the count pins exactly; the average is
    printed to one decimal, so it pins the sum of seed lengths to within 0.05 per seed"""
    c = pc.case(name)
    ref = pc.reference_merge(c)
    ps = c.pstart2()
    for f in c.freqs:
        s, sl = ol.merge(c.T1, c.T2, ps, f)
        r = ref[str(f)]
        assert len(s) == r["seeds"], f
        if len(s):
            assert abs(sl / len(s) - r["avelen"]) <= 0.05 + 1e-9, f

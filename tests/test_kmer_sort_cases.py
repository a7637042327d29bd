"""The crafted inputs of kmer_sort_cases.py without a GPU: every case reaches the edges of the k-mer sort and the
syncmer scan it is named for, by the numpy restatements of their rules; together the cases reach every row of
the regime table; record cases keep the input contract of fgb_gix_from_records; the restated sampler histogram
and the restated records per scan tile agree with the oracle."""
import functools

import numpy as np
import pytest

import kmer_sort_cases as kc
import oracle_lib as ol

#  what each case is named for: the rows of kmer_sort_cases.ROWS it must reach
REACH = {
    "plan_bins_0_1_cap-1_cap": {"bin_0", "bin_1", "bin_cap-1", "bin_cap"},
    "plan_bin_cap+1": {"bin_cap+1", "over1", "over_slot1", "ototal=tile+1"},
    "plan_window_sums_cap_cap+1": {"window_cap", "window_cap+1", "bin_0"},
    "plan_oversized_slots_0_1_2_3": {"over_slot0", "over_slot1", "over_flush", "over_slot3", "over3+",
                                     "over_random", "over_lsd_fast", "ototal>2tiles"},
    "plan_nbins_mod4_1": {"nbins%4=1", "passes3"}, "plan_nbins_mod4_2": {"nbins%4=2", "passes3"},
    "plan_nbins_mod4_3": {"nbins%4=3", "passes3"},
    "plan_nbins_1": {"nbins=1", "one_digit_first"},
    "plan_one_bin_of_65536": {"one_bin_of_65536", "one_digit_first", "passes2"},
    "share_unaligned_plo_phi": {"plo_unaligned", "phi_unaligned"},
    "share_first_bin_only": {"first_bin_only", "plo_unaligned"},
    "share_last_bin_only": {"last_bin_only", "phi_unaligned"},
    "share_phi_top": {"phi_top"},
    "share_empty_ends": {"empty_ends"},
    "sub_31_32_33": {"sub31", "sub32", "sub33", "tie_post_fast", "tie_strand_fast", "tie_contig_fast",
                     "tie_byte0_lsd"},
    "sub_lo_ties_fast_and_lsd": {"tie_strand_fast", "tie_contig_fast", "tie_post_fast", "tie_lo16_fast",
                                 "tie_strand_lsd", "tie_contig_lsd", "tie_post_lsd", "tie_lo16_lsd"},
    "sub_crowded_in_each_bin": {"crowded_each_bin"},
    "cta_loop_fast_lsd_alternating": {"cta_loop3", "cta_mixed"},
    "over_two_descending_lsd_fast": {"over2", "over_desc", "over_lsd_fast", "ototal>2tiles"},
    "over_three_ascending": {"over3+", "over_asc"},
    "over_last_bin_two_tiles": {"over1", "over_last", "ototal=2tiles"},
    "over_300_random": {"over300", "over_random"},
    "part_n0": {"n=0"}, "part_n1": {"n=1"}, "part_n2": {"n=2"}, "part_n4095": {"n=tile-1"},
    "part_n4096": {"n=tile"}, "part_n4097": {"n=tile+1"}, "part_n8193": {"n=2tile+1"},
    "part_one_first_digit": {"one_digit_first"},
    "part_target1_3passes_131072_bins": {"passes3", "bins>65536"},
    "part_target1_2passes": {"passes2"},
    "scan_stage_both": {"tile=stage_both", "tile=stage+1_both", "rounds4", "rounds4_contig_end", "width8",
                        "sh-fsh=0"},
    "scan_stage_fwd": {"tile=stage_fwd", "tile=stage+1_fwd", "rounds4"},
    "scan_digit9_both": {"width9", "sh-fsh=1", "scan_passes1"},
    "scan_digit9_fwd": {"width9", "sh-fsh=1"},
    "scan_range_fsh3_sh6": {"sh-fsh=2+", "scan_passes2"},
    "scan_range_top_unaligned": {"sh-fsh=2+"},
}
REACH.update({"scan_range_fsh%d" % k: {"width%d" % w, "sh-fsh=0"}
              for k, w in enumerate((8, 7, 6, 5, 4, 3, 2, 9))})

ALL_ROWS = [r for rows in kc.ROWS.values() for r in rows]


@functools.lru_cache(maxsize=None)
def _oracle(which):
    c = next(kc.genome_case(n) for n in kc.GENOME_NAMES if kc._genome_cases()[n][0] == which)
    rank = ol.contig_rank([len(s) for s in c.contigs])[1]
    return ol.gix_build(c.genome, rank)[0], rank


@functools.lru_cache(maxsize=None)
def _rows(name):
    if name in kc.RECORD_NAMES:
        return frozenset(kc.record_rows(kc.record_case(name)))
    c = kc.genome_case(name)
    return frozenset(kc.genome_rows(c, *_oracle(kc._genome_cases()[name][0])))


def test_every_case_states_its_edges():
    assert sorted(REACH) == sorted(kc.RECORD_NAMES + kc.GENOME_NAMES)
    assert set().union(*REACH.values()) <= set(ALL_ROWS)


@pytest.mark.parametrize("name", kc.RECORD_NAMES + kc.GENOME_NAMES)
def test_case_reaches_its_edges(name):
    missing = REACH[name] - _rows(name)
    assert not missing, missing


def test_every_row_is_reached():
    by_row = {r: [] for r in ALL_ROWS}
    for name in kc.RECORD_NAMES + kc.GENOME_NAMES:
        for r in _rows(name):
            by_row.setdefault(r, []).append(name)
    for group, rows in kc.ROWS.items():
        print("%s:" % group)
        for r in rows:
            print("  %-20s %s" % (r, " ".join(by_row[r])))
    assert [r for r in ALL_ROWS if not by_row[r]] == []


@pytest.mark.parametrize("name", kc.RECORD_NAMES)
def test_record_case_keeps_the_input_contract(name):
    """prefixes in [plo, phi), every record unique: outside the range the fine-bin and sub-bin arithmetic of the
    sort wraps"""
    c = kc.record_case(name)
    r = c.records
    assert r.dtype == np.uint64 and r.ndim == 2 and r.shape[1] == 2
    pre = r[:, 1] >> np.uint64(40)
    assert ((pre >= c.plo) & (pre < c.phi)).all()
    assert 0 <= c.plo < c.phi <= kc.TOP
    assert len(np.unique(r, axis=0)) == len(r)


def test_restated_rules_at_their_edges():
    """bin_shift and first_digit at the switch points of their rules"""
    T = kc.TOP
    assert kc.bin_shift(0, 0, T) == 8 and kc.bin_shift(1537 * 65536 - 1, 0, T) == 8
    assert kc.bin_shift(1537 * 65536, 0, T) == 7
    assert kc.bin_shift(2 * 65536 - 1, 0, T, 1) == 8 and kc.bin_shift(2 * 65536, 0, T, 1) == 7
    assert kc.bin_shift(2 * 65536, 0, T, 0) == 7 and kc.bin_shift(4 * 65536 - 1, 0, T, 1) == 7
    assert kc.bin_shift(4 * 65536, 0, T, 1) == 6
    assert kc.bin_shift(5, 7, 8) == 0 and kc.bin_shift(5, 0, 65536) == 0 and kc.bin_shift(5, 0, 65537) == 1
    assert kc.bin_shift(5, 1, 65537) == 0 and kc.bin_shift(5, 1, 65538) == 1      # a share's partial bins
    widths = {fsh: kc.first_digit(0, 0, 1 << (16 + fsh)) for fsh in range(9)}
    assert widths == {0: (0, 8), 1: (1, 7), 2: (2, 6), 3: (3, 5), 4: (4, 4), 5: (5, 3), 6: (6, 2), 7: (7, 9),
                      8: (8, 8)}


def test_plan_groups_on_crafted_bins():
    C = kc.BK_CAP
    sizes = [1, 0, 2, 0, C - 1, 0, 0, 0, C, 0, 0, 0, 5, C + 1, 9, 0, 1000, 1000, 1000, C - 2999, 20, 200, 6000, 50,
             3]
    bins = np.concatenate([[0], np.cumsum(sizes)])
    groups, over = kc.plan_groups(bins)
    b = [int(x) for x in bins]
    assert groups == [(0, 3, 0), (b[4], C - 1, 4), (b[8], C, 8), (b[12], 5, 12), (b[14], 9, 14),
                      (b[16], 3000, 16), (b[19], C - 2999, 19), (b[20], 220, 20), (b[23], 50, 23), (b[24], 3, 24)]
    assert over == [(b[13], C + 1), (b[22], 6000)]


@pytest.mark.parametrize("which", ["stage_both", "stage_fwd", "random"])
def test_restatements_agree_with_the_oracle_table(which):
    """the records per scan tile (from orc_syncmers) are the oracle table's records by tile; the sampler histogram
    (from orc_syncmers and the bases) is the first five bases of the oracle's both-strand entries, plus those of
    the sampled positions near a contig end that give no forward or no reverse entry"""
    tab, rank = _oracle(which)
    contigs = kc._contigs(which)
    c = kc.GenomeCase(which, contigs, "both")
    tile, ntiles = kc.tile_of(c, tab, rank)
    fwd = (tab[:, 0] >> np.uint64(47)) & np.uint64(1) == 0
    for fwd_only in (False, True):
        want = np.concatenate([kc.tile_records(s, fwd_only) for s in contigs if len(s) >= 12])
        assert np.array_equal(np.bincount(tile[fwd] if fwd_only else tile, minlength=ntiles), want)
    h = np.bincount((tab[:, 1] >> np.uint64(54)).astype(np.int64), minlength=1024)
    for s in contigs:
        pos = kc.syncmers(s)
        s = np.asarray(s, dtype=np.int64)
        nf, nr = pos[pos > len(s) - 40], pos[pos < 28]
        h += np.bincount(sum(s[nf + k] << (2 * (4 - k)) for k in range(5)), minlength=1024)
        h += np.bincount(sum((3 - s[nr + 11 - k]) << (2 * (4 - k)) for k in range(5)), minlength=1024)
    assert np.array_equal(kc.buck1024(contigs), h)
    assert kc.buck1024(contigs).sum() == 2 * sum(len(kc.syncmers(s)) for s in contigs)

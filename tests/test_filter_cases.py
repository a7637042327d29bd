"""CPU tests of the redundancy filter and the final .1aln order: the product's fgb_filter
(fastga_b200/csrc/filter.cu) against the oracle's orc_filter (oracle/fastga_oracle.c, written after
FastGA.c:2818-2941, :3405-3685 and :3800-3835), field by field, trace byte by trace byte, in output
order.  Crafted groups (tests/filter_cases.py) each reach the branch they are named for; a seeded
random corpus of groups cut from a few shared paths reaches every branch; the raw records of the
oracle's own search on real inputs go through both filters as well.

What real data reaches (oracle search, default parameters): small_pair and the SELF genomes dup and
tandem61 together reach same-start-and-end drops with o kept (75), B-disjoint skips (9), box drops of
w (201) and of o (182) and apart-and-kept pairs (197); they reach no other sweep-1 outcome, no fusion
and no crossing, which only the crafted cases and the corpus exercise."""
import numpy as np
import pytest

import filter_cases as fc
import oracle_lib as ol
from fastga_b200 import formats, synth


@pytest.mark.parametrize("name", sorted(fc.CASES))
def test_crafted_case_reaches_its_counter_and_filters_agree(name):
    build, want = fc.CASES[name]
    case = build()
    got, cnt = fc.run_oracle(case)
    assert fc.counters_reached(cnt, want), (want, cnt)
    prod = fc.run_product(case)
    assert fc.differences(prod, got) == ""
    shuffled = fc.run_product(case, shuffle_seed=len(name))
    assert fc.differences(shuffled, got) == ""


def test_crafted_outcomes():
    """what each rule leaves, spelled out where a kernel is most easily wrong"""
    al, _ = fc.run_oracle(fc.same_both_drop_o())
    assert len(al) == 1 and al.fields[0, 7] == 7                 # o (diffs 450 >= aepos 450) went
    al, _ = fc.run_oracle(fc.same_both_diffs_at_aepos_minus_1())
    assert len(al) == 1 and al.fields[0, 7] == 449
    al, _ = fc.run_oracle(fc.fuse())                              # cut at 400, the last meet: 4 + 4 intervals
    assert len(al) == 1 and al.fields[0, 3:9].tolist() == [0, 1000, 800, 1800, 1 + 2 + 3 + 4 + 7 + 6 + 5 + 4, 16]
    al, _ = fc.run_oracle(fc.several_meets_last_wins())
    assert len(al) == 1 and al.trace(0)[0::2].tolist() == [1, 1, 1, 1, 1, 9, 9, 9]
    assert al.trace(0)[1::2].tolist() == [100] * 5 + [103, 100, 100]
    al, _ = fc.run_oracle(fc.fuse_into_dead_o())                  # o fused but dead: w1 alone is left
    assert len(al) == 1 and al.fields[0, 3] == 5
    al, _ = fc.run_oracle(fc.row_extended_boxes_in())           # x dropped only by the re-read row
    assert len(al) == 1 and al.fields[0, 3:7].tolist() == [0, 1000, 1000, 2000]
    for nm, n in (("truncation_decides_sign", 2), ("truncation_keeps_apart", 1),
                  ("k_on_grid_point_meets_only_there", 2), ("zero_only_at_end", 2)):
        al, _ = fc.run_oracle(fc.CASES[nm][0]())
        assert len(al) == n, nm


def test_sort_map_keys():
    """(aread, abpos, bread, comp), then the position in the filter's output"""
    al, _ = fc.run_oracle(fc.sort_map_comp_before_position())
    assert al.fields[:, :3].tolist() == [[0, 0, 0], [0, 0, 1], [1, 0, 1], [0, 1, 0]]
    al, _ = fc.run_oracle(fc.sort_map_full_ties())
    assert al.fields[:, [0, 2, 5]].tolist() == [[0, 0, 900], [0, 0, 700], [0, 0, 1400], [1, 0, 600], [1, 0, 900],
                                                [0, 1, 800]]


def test_fuzz_edges_flip_at_eleven():
    for side in ("w", "o"):
        for e in (("aepos", "bbpos", "bepos") if side == "w" else ("abpos", "bbpos", "bepos")):
            a10, _ = fc.run_oracle(fc.CASES["fuzz_drop_%s_%s_10" % (side, e)][0]())
            a11, _ = fc.run_oracle(fc.CASES["fuzz_drop_%s_%s_11" % (side, e)][0]())
            assert (len(a10), len(a11)) == (1, 2), (side, e)


@pytest.mark.parametrize("n", [2, 3, 17, 100, 1000])
def test_abpos_ties_keep_qsort_order(n):
    """records that tie on abpos and all survive: their .1aln order is the sweep's qsort tie order"""
    case = fc.abpos_ties(n, n)
    got, _ = fc.run_oracle(case)
    assert len(got) == n - (n - 1) // 5 and (got.fields[:, 3] == 500).all()
    assert fc.differences(fc.run_product(case), got) == ""


def test_do_filter_0_keeps_every_record_in_order():
    for case in (fc.interleaved_groups(), fc.interleaved_groups(True, 8), fc.corpus(3)):
        got, cnt = fc.run_oracle(case, do_filter=False)
        assert len(got) == sum(len(g[3]) for g in case["groups"]) and not any(cnt.values())
        assert fc.differences(fc.run_product(case, do_filter=False, shuffle_seed=1), got) == ""


def test_random_corpus_agrees_and_lights_every_counter():
    total = dict.fromkeys(ol.FILTER_COUNTERS, 0)
    for seed in range(40):
        case = fc.corpus(seed)
        got, cnt = fc.run_oracle(case)
        for k, v in cnt.items():
            total[k] += v
        d = fc.differences(fc.run_product(case, shuffle_seed=seed), got)
        assert d == "", (seed, d)
    print("corpus counters", total)
    assert all(v > 0 for v in total.values()), total


def _real_inputs():
    A, B = synth.make_pair(11, 1_200_000, 3, 0.05, sv_every=60000)
    yield "small_pair", ol.oracle_pipeline(formats.genome_from_arrays(A), formats.genome_from_arrays(B))
    import test_oracle_pin
    G = test_oracle_pin._self_genomes()
    for nm in ("dup", "tandem61"):
        yield nm, ol.oracle_pipeline_self(formats.genome_from_arrays(G[nm]))


def test_real_raw_groups_agree():
    """every raw group of the oracle's search on small_pair and two SELF genomes through both filters"""
    total = dict.fromkeys(ol.FILTER_COUNTERS, 0)
    for nm, r in _real_inputs():
        assert fc.differences(r["alns_product"], r["alns"]) == "", nm
        for k, v in r["filter_counters"].items():
            total[k] += v
    print("real-data counters", total)
    assert total["s1_same_keep_o"] > 0 and total["s2_b_disjoint"] > 0

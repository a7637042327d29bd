"""Crafted raw alignment groups for the redundancy filter and the final .1aln order (fgb_filter against
the oracle's orc_filter, tests/test_filter_cases.py).

A record is built from its start point, one B-advance per trace interval and one diffs byte per
interval (rec()): the trace is consistent by construction and bepos = bbpos + the B-advances.  A case is
a list of groups, each the raw output of one align_contigs call: (comp, aread, bread, records in
discovery order), plus the contig ranks that map contig numbers to the seed records' contig fields.
CASES maps a case name to (builder, the filter counters it must reach).  run_oracle() and
run_product() put one case through either filter; corpus() makes the seeded random groups."""
import numpy as np

import oracle_lib as ol

TSPACE = 100


def rec(ab, bb, badv, diffs=None, ae=None):
    """one raw record: starts at (ab, bb), B-advances badv per trace interval; ends at ae (default: the
    grid point after the last full interval, or ab + 100 * intervals when ab lies on the grid)"""
    n = len(badv)
    if ae is None:
        ae = (ab // TSPACE + n) * TSPACE
    assert (ae - 1) // TSPACE - ab // TSPACE + 1 == n, "intervals of [%d, %d] != %d" % (ab, ae, n)
    if diffs is None:
        diffs = [0] * n
    elif np.isscalar(diffs):
        diffs = [int(diffs)] * n
    assert len(diffs) == n and all(0 <= int(v) <= 255 for v in list(badv) + list(diffs))
    tr = np.empty(2 * n, dtype=np.uint8)
    tr[0::2] = diffs
    tr[1::2] = badv
    return dict(ab=int(ab), bb=int(bb), ae=int(ae), be=int(bb + sum(int(v) for v in badv)),
                diffs=int(sum(int(v) for v in diffs)), trace=tr)


def diag(ab, ae, bb, diffs=None):
    """a record on one diagonal: B advances as much as A in every interval"""
    pts = [ab] + list(range((ab // TSPACE + 1) * TSPACE, ae, TSPACE)) + [ae]
    return rec(ab, bb, [pts[i + 1] - pts[i] for i in range(len(pts) - 1)], diffs, ae)


def one(*recs, comp=0, aread=0, bread=0):
    """a case of one group"""
    return dict(groups=[(comp, aread, bread, list(recs))], nA=max(aread + 1, 1), nB=max(bread + 1, 1))


# ------------------------------------------------------------------------------------------------
#  running one case through both filters
# ------------------------------------------------------------------------------------------------

def _flat(case):
    """the records in discovery order with their group index"""
    out = []
    for g, (comp, ar, br, recs) in enumerate(case["groups"]):
        for r in recs:
            out.append((g, comp, ar, br, r))
    return out


def run_oracle(case, do_filter=True):
    """orc_filter on the case: (lib.Alignments, counters)"""
    flat = _flat(case)
    ov = np.zeros(len(flat), dtype=ol.OVL_DT)
    pool, off = [], 0
    for i, (g, comp, ar, br, r) in enumerate(flat):
        ov[i] = (comp, ar, br, r["ab"], r["bb"], r["ae"], r["be"], r["diffs"], len(r["trace"]), g, off)
        pool.append(r["trace"])
        off += len(r["trace"])
    tp = np.concatenate(pool) if pool else np.zeros(0, np.uint8)
    al = ol.filter(ov, tp, do_filter)
    return al, ol.filter_counters()


def _ranks(case):
    nA, nB = case["nA"], case["nB"]
    r1 = np.asarray(case.get("rank1", np.arange(nA)), dtype=np.int32)
    r2 = r1 if case.get("self") else np.asarray(case.get("rank2", np.arange(nB)), dtype=np.int32)
    return r1, r2


def run_product(case, do_filter=True, shuffle_seed=None, per_triple=3):
    """fgb_filter on the case, the records packed as the extension emits them: (triple, seq) give the
    discovery order (per_triple records per triple), the buffer itself is shuffled when shuffle_seed is
    set"""
    from fastga_b200 import lib
    flat = _flat(case)
    r1, r2 = _ranks(case)
    jb = max(int(max(case["nB"] - 1, 1)).bit_length(), 1)
    ib = max(int(max(case["nA"] - 1, 1)).bit_length(), 1)
    parts = []
    for i, (g, comp, ar, br, r) in enumerate(flat):
        pk = (comp << (jb + ib)) | (int(r1[ar]) << jb) | int(r2[br])
        h = np.array([i // per_triple, i % per_triple, pk, r["ab"], r["bb"], r["ae"], r["be"], r["diffs"],
                      len(r["trace"]), 0], dtype=np.int32)
        tr = r["trace"].tobytes()
        parts.append(h.tobytes() + tr + b"\0" * ((-len(tr)) % 8))
    if shuffle_seed is not None:
        np.random.default_rng(shuffle_seed).shuffle(parts)
    buf = np.frombuffer(b"".join(parts), dtype=np.uint8) if parts else np.zeros(0, np.uint8)
    O = lib.overlaps_from_buffer(buf)
    p1 = np.argsort(r1).astype(np.int32)
    p2 = p1 if case.get("self") else np.argsort(r2).astype(np.int32)
    return lib.filter_overlaps(O.h, p1, p2, jb, ib, do_filter)


differences = ol.alignment_differences


# ------------------------------------------------------------------------------------------------
#  sweep 1: equal start points, equal end points
# ------------------------------------------------------------------------------------------------

def same_both_keep_o():
    # equal ends: o survives while its diffs are below w's aepos (FastGA.c:3456 compares them)
    return one(diag(0, 450, 1000, [3, 1, 0, 2, 5]), diag(0, 450, 1000, [1, 1, 1, 1, 1]))


def same_both_drop_o():
    # o.diffs = 450 = w.aepos: not below, so o goes and w stays
    return one(diag(0, 450, 1000, [100, 100, 100, 100, 50]), diag(0, 450, 1000, [7, 0, 0, 0, 0]))


def same_both_diffs_at_aepos_minus_1():
    # o.diffs = 449 < 450: o stays
    return one(diag(0, 450, 1000, [100, 100, 100, 100, 49]), diag(0, 450, 1000, [7, 0, 0, 0, 0]))


def same_start_keep_o():
    # discovery order long, short: qsort keeps the tie's order, o is the longer one
    return one(diag(200, 900, 1000), diag(200, 640, 1000, 2))


def same_start_drop_o():
    # short first: o ends before w, so o goes and its row ends
    return one(diag(200, 640, 1000, 2), diag(200, 900, 1000))


def same_start_equal_aepos():
    # same start, same aepos, different bepos: not `o.aepos > w.aepos`, o goes
    return one(diag(200, 640, 1000), rec(200, 1000, [100, 100, 100, 100, 45]))


def same_end_keep_o():
    return one(diag(130, 900, 1130), diag(400, 900, 1400, 1))


def same_end_drop_o():
    # equal abpos, different bbpos, same end: o does not start before w, so o goes
    return one(rec(300, 1000, [100, 100, 100, 100, 100]), rec(300, 990, [110, 100, 100, 100, 100]))


def dead_o_in_sweep_one_keeps_no_w_alive():
    # o dies in its row at the first w that shares its end; a later w sharing its start survives
    return one(diag(300, 800, 1300), diag(300, 800, 1300, 9), diag(400, 1200, 1400))


# ------------------------------------------------------------------------------------------------
#  sweep 2
# ------------------------------------------------------------------------------------------------

def b_disjoint():
    return one(diag(0, 800, 1000), diag(300, 900, 5000))


def fuse():
    # same diagonal, distinct ends: they meet at 300 and 400, the last one is the cut
    return one(diag(0, 500, 1000, [1, 2, 3, 4, 5]), diag(250, 800, 1250, [9, 8, 7, 6, 5, 4]))


def fuse_into_dead_o():
    # o is boxed in by the longer w1 (5 above, parallel), finishes its row and still absorbs w2
    return one(diag(0, 400, 1000, 1), diag(5, 700, 1010, 2), diag(200, 900, 1200, 3))


def fuse_w_owns_trace():
    # w fuses with x in its own row first, then o fuses with the fused w
    return one(diag(0, 400, 1000, 1), diag(200, 700, 1200, 2), diag(500, 1000, 1500, 3))


def box_drop_w():
    return one(diag(0, 1000, 1000), diag(300, 600, 1303))


def box_drop_o():
    return one(diag(0, 300, 1000), diag(5, 1000, 1008))


def apart_kept():
    return one(diag(0, 500, 1000), diag(300, 900, 1303))


def cross():
    # w starts 5 above o's path and ends 5 below it; no trace point at separation 0
    return one(diag(0, 600, 1000), rec(250, 1255, [50, 90, 100], ae=500))


def row_extended():
    # the fusion at 300 moves o's end from 400 to 900: o's row then reaches x at 450
    return one(diag(0, 400, 1000), diag(200, 900, 1200), diag(450, 600, 5000))


def row_extended_boxes_in():
    # the fusion at 300 gives o w's end (1000) and keeps o's start: x at 450, flat and below w's B start,
    # is B-disjoint from w in w's row but inside the fused o's box in o's re-read row
    return one(diag(0, 400, 1000), diag(200, 1000, 1200), rec(450, 1100, [10, 20, 20], ae=700))


# ------------------------------------------------------------------------------------------------
#  BOX_FUZZ edges, the length test
# ------------------------------------------------------------------------------------------------

def _fuzz_drop_w(edge, f):
    o = diag(0, 1000, 1000)
    if edge == "aepos":                               # w ends f past o, 3 below it
        w = diag(500, 1000 + f, 1497)
    elif edge == "bbpos":                             # w starts f below o's bbpos
        w = diag(200, 800, 1000 - f)
    else:                                             # bepos: w ends f above o's bepos
        w = diag(200, 800, 1400 + f)
    return one(o, w)


def _fuzz_drop_o(edge, f):
    o = diag(100, 500, 1100)
    if edge == "abpos":                               # w starts f after o, 3 below it
        w = diag(100 + f, 1500, 1097 + f)
    elif edge == "bbpos":                             # o starts f below w's bbpos
        w = diag(105, 1500, 1100 + f)
    else:                                             # bepos: o ends f above w's bepos, w runs flatter
        n = 14
        adv = [36] * n
        adv[-1] = (500 - f) - 36 * (n - 1)
        w = rec(105, 1000, adv, ae=1500)
    return one(o, w)


def len_w_is_len_o_plus_10():
    # w (same abpos, 3 below) is 10 longer: still o's box test, and w is inside it
    return one(diag(0, 500, 1000), diag(0, 510, 997))


def len_w_is_len_o_plus_11():
    # 11 longer: w's box test, and o is inside it
    return one(diag(0, 500, 1000), diag(0, 511, 997))


# ------------------------------------------------------------------------------------------------
#  entwine's geometry
# ------------------------------------------------------------------------------------------------

def same_interval_short_k():
    # K starts in J's first interval and is under one interval long: one separation at K's start, one
    # at its end interpolated from the trace point at 100 (not from K's start), 1 above: boxed in
    return one(diag(110, 600, 1110), rec(130, 1133, [50], ae=180))


def same_interval_short_k_touching():
    # the same, 2 above: the end separation interpolates to 0 -- touching, no action
    return one(diag(110, 600, 1110), rec(130, 1132, [50], ae=180))


def k_on_grid_point_meets_only_there():
    # K starts on the grid at separation 0, then runs 2 above: its start is no meeting point
    return one(diag(0, 800, 1000), rec(300, 1300, [102, 100, 100], ae=600))


def k_on_grid_point_fuses():
    return one(diag(0, 800, 1000, 2), diag(300, 1100, 1300, 1))


def zero_only_at_end():
    # separations 3, 2, 1 at the trace points and 0 only at o's end: no meet, the paths touch
    return one(diag(0, 400, 1000), rec(150, 1153, [49, 99, 99, 100], ae=500))


def several_meets_last_wins():
    # the paths meet at 300 and at 500 (2 apart at 400, 3 apart from 600 on): the cut is at 500
    o = diag(0, 700, 1000, [1, 1, 1, 1, 1, 1, 1])
    w = rec(250, 1250, [50, 102, 98, 103, 100, 100], diffs=[9, 9, 9, 9, 9, 9], ae=800)
    return one(o, w)


def wide_b_advances():
    # B-advances of 128 and more on both paths (unsigned bytes): a fusion on a steep shared path
    adv = [200, 180, 255, 128, 140, 250, 129, 131]
    bpos = np.concatenate([[0], np.cumsum(adv)])
    o = rec(0, 1000, adv[:5], [1] * 5)
    w = rec(200, 1000 + int(bpos[2]), adv[2:], [2] * 6)
    return one(o, w)


def wide_b_advances_apart():
    adv = [200, 180, 255, 128, 140, 250, 129, 131]
    o = rec(0, 1000, adv[:6], [1] * 6)
    w = rec(100, 1000 + 200 + 7, adv[1:5], [2] * 4)
    return one(o, w)


def truncation_decides_sign():
    # o advances 99 in [200, 300): at K's start 250 the interpolation is 49.5, truncated to 49, so the
    # start separation is 0 while every other one is -1: touching (no action).  Rounding would make
    # them all -1 and box w in.
    o = rec(0, 1000, [100, 100, 99, 100, 100, 100], ae=600)
    w = rec(250, 1000 + 200 + 49, [49, 100, 100], ae=500)
    return one(o, w)


def truncation_keeps_apart():
    # o advances 99 in [200, 300) and w starts at 251: 99 * 51 / 100 = 50.49 -> 50, separation -1 with
    # every other one -1: apart, boxed in
    o = rec(0, 1000, [100, 100, 99, 100, 100, 100], ae=600)
    w = rec(251, 1000 + 200 + 49, [49, 100, 100], ae=500)
    return one(o, w)


# ------------------------------------------------------------------------------------------------
#  ties and the final order
# ------------------------------------------------------------------------------------------------

def abpos_ties(n, seed=0):
    """n records with one abpos on B-disjoint paths of random lengths: none is dropped, so the
    output order is the qsort tie order; every fifth one shares its start with the one before"""
    rng = np.random.default_rng(seed)
    recs = []
    for i in range(n):
        ln = int(rng.integers(1, 12)) * 100 + int(rng.integers(0, 100))
        bb = 10_000 * i + 1000 if i % 5 else 10_000 * (i - 1) + 1000 if i else 1000
        recs.append(diag(500, 500 + ln, bb, int(rng.integers(0, 5))))
    return one(*recs)


def interleaved_groups(self_mode=False, seed=7):
    """several (A, B, strand) groups, contig ranks that are not the identity, records of one group
    spread over many triples, and SORT_MAP ties: equal (aread, abpos) across B contigs and strands"""
    rng = np.random.default_rng(seed)
    nA, nB = 5, 5 if self_mode else 4
    groups = []
    for comp in (0, 1):
        for ar in (3, 0, 4):
            for br in ((1, 3, 0) if not self_mode else (3, 0, 2)):
                recs = []
                for k in range(int(rng.integers(1, 7))):
                    ab = int(rng.choice([100, 100, 250, 1000, 1333]))
                    ln = int(rng.integers(2, 15)) * 100
                    off = int(rng.choice([0, 0, 4, 30_000]))
                    recs.append(diag(ab, ab + ln, 2000 + ab + off + 100_000 * k, int(rng.integers(0, 4))))
                if rng.random() < 0.5:                      # a duplicate to drop
                    recs.append(dict(recs[0]))
                groups.append((comp, ar, br, recs))
    rank1 = np.array([2, 4, 0, 1, 3], np.int32)
    case = dict(groups=groups, nA=nA, nB=nB, rank1=rank1, rank2=np.array([3, 0, 2, 1], np.int32))
    if self_mode:
        case["self"] = True
    return case


def sort_map_full_ties():
    """records that agree on (aread, abpos, bread, comp) survive side by side in one group (apart in B)
    and across the two strands of the same contig pair: position decides"""
    g0 = [diag(500, 900, 1000), diag(500, 700, 9000), diag(500, 1400, 20_000)]
    g1 = [diag(500, 600, 3000), diag(500, 900, 4000)]
    return dict(groups=[(0, 1, 0, g0), (0, 1, 1, [diag(500, 800, 7000)]), (1, 1, 0, g1)], nA=2, nB=2,
                rank1=np.array([1, 0], np.int32), rank2=np.array([1, 0], np.int32))


def sort_map_comp_before_position():
    """a strand-C group found before the strand-N group of the same contig pair, both starting at the
    same abpos: the strand, not the position, puts the N record first"""
    return dict(groups=[(1, 0, 1, [diag(500, 900, 1000)]), (0, 0, 1, [diag(500, 700, 3000)]),
                        (0, 1, 0, [diag(500, 800, 3000)]), (0, 0, 0, [diag(500, 600, 3000)])], nA=2, nB=2)


# ------------------------------------------------------------------------------------------------
#  the table: case -> (builder, counters it must reach)
# ------------------------------------------------------------------------------------------------

CASES = {
    "same_both_keep_o": (same_both_keep_o, {"s1_same_keep_o": 1}),
    "same_both_drop_o": (same_both_drop_o, {"s1_same_drop_o": 1}),
    "same_both_diffs_at_aepos_minus_1": (same_both_diffs_at_aepos_minus_1, {"s1_same_keep_o": 1}),
    "same_start_keep_o": (same_start_keep_o, {"s1_start_keep_o": 1}),
    "same_start_drop_o": (same_start_drop_o, {"s1_start_drop_o": 1}),
    "same_start_equal_aepos": (same_start_equal_aepos, {"s1_start_drop_o": 1}),
    "same_end_keep_o": (same_end_keep_o, {"s1_end_keep_o": 1}),
    "same_end_drop_o": (same_end_drop_o, {"s1_end_drop_o": 1}),
    "dead_o_in_sweep_one": (dead_o_in_sweep_one_keeps_no_w_alive, {"s1_same_drop_o": 0, "s1_same_keep_o": 1}),
    "b_disjoint": (b_disjoint, {"s2_b_disjoint": 1}),
    "fuse": (fuse, {"s2_fuse": 1}),
    "fuse_into_dead_o": (fuse_into_dead_o, {"s2_box_drop_o": 1, "s2_fuse_dead_o": 1}),
    "fuse_w_owns_trace": (fuse_w_owns_trace, {"s2_fuse": 2, "s2_fuse_w_owns": 1}),
    "box_drop_w": (box_drop_w, {"s2_box_drop_w": 1}),
    "box_drop_o": (box_drop_o, {"s2_box_drop_o": 1}),
    "apart_kept": (apart_kept, {"s2_apart_kept": 1}),
    "cross": (cross, {"s2_cross": 1}),
    "row_extended": (row_extended, {"s2_fuse": 1, "s2_row_extended": 1}),
    "row_extended_boxes_in": (row_extended_boxes_in, {"s2_fuse": 1, "s2_row_extended": 1, "s2_box_drop_w": 1}),
    "len_w_is_len_o_plus_10": (len_w_is_len_o_plus_10, {"s2_box_drop_w": 1}),
    "len_w_is_len_o_plus_11": (len_w_is_len_o_plus_11, {"s2_box_drop_o": 1}),
    "same_interval_short_k": (same_interval_short_k, {"s2_box_drop_w": 1}),
    "same_interval_short_k_touching": (same_interval_short_k_touching, {"s2_cross": 1}),
    "k_on_grid_point_meets_only_there": (k_on_grid_point_meets_only_there, {"s2_cross": 1}),
    "k_on_grid_point_fuses": (k_on_grid_point_fuses, {"s2_fuse": 1}),
    "zero_only_at_end": (zero_only_at_end, {"s2_cross": 1}),
    "several_meets_last_wins": (several_meets_last_wins, {"s2_fuse": 1}),
    "wide_b_advances": (wide_b_advances, {"s2_fuse": 1}),
    "wide_b_advances_apart": (wide_b_advances_apart, {"s2_box_drop_w": 1}),
    "truncation_decides_sign": (truncation_decides_sign, {"s2_cross": 1}),
    "truncation_keeps_apart": (truncation_keeps_apart, {"s2_box_drop_w": 1}),
    "sort_map_full_ties": (sort_map_full_ties, {"s2_b_disjoint": 2}),
    "sort_map_comp_before_position": (sort_map_comp_before_position, {}),
    "interleaved_groups": (interleaved_groups, {"s1_same_keep_o": 1}),
    "interleaved_groups_self": (lambda: interleaved_groups(True, 8), {"s1_same_keep_o": 1}),
}
for _e in ("aepos", "bbpos", "bepos"):
    CASES["fuzz_drop_w_%s_10" % _e] = ((lambda e=_e: _fuzz_drop_w(e, 10)), {"s2_box_drop_w": 1})
    CASES["fuzz_drop_w_%s_11" % _e] = ((lambda e=_e: _fuzz_drop_w(e, 11)), {"s2_box_drop_w": 0, "s2_apart_kept": 1})
for _e in ("abpos", "bbpos", "bepos"):
    CASES["fuzz_drop_o_%s_10" % _e] = ((lambda e=_e: _fuzz_drop_o(e, 10)), {"s2_box_drop_o": 1})
    CASES["fuzz_drop_o_%s_11" % _e] = ((lambda e=_e: _fuzz_drop_o(e, 11)), {"s2_box_drop_o": 0, "s2_apart_kept": 1})
for _n in (2, 3, 17, 100, 1000):
    CASES["abpos_ties_%d" % _n] = ((lambda n=_n: abpos_ties(n, n)), {"s1_start_keep_o": 0} if _n == 2 else {})


def counters_reached(got, want):
    """want: counter -> n; n > 0 asks for at least n, 0 for none"""
    return all((got[k] >= v) if v else (got[k] == 0) for k, v in want.items())


# ------------------------------------------------------------------------------------------------
#  the seeded random corpus
# ------------------------------------------------------------------------------------------------

def _shared_path(rng, length):
    """B position at every trace point of a path over A [0, length]"""
    steps = rng.integers(70, 140, length // TSPACE + 2)
    steps[rng.random(len(steps)) < 0.05] = rng.integers(128, 256)
    return np.concatenate([[0], np.cumsum(steps)]).astype(np.int64)


def _b_at(path, a):
    g = a // TSPACE
    return int(path[g] + ((path[g + 1] - path[g]) * (a - g * TSPACE)) // TSPACE)


def _cut(rng, path, base, a, e, off):
    """the piece [a, e] of a shared path, shifted by off in B, one interval bent by +-1 now and then"""
    pts = [a] + list(range((a // TSPACE + 1) * TSPACE, e, TSPACE)) + [e]
    bs = [_b_at(path, p) for p in pts]
    adv = [bs[i + 1] - bs[i] for i in range(len(pts) - 1)]
    if len(adv) >= 3 and rng.random() < 0.15:
        i = int(rng.integers(0, len(adv) - 1))
        if adv[i] < 255 and adv[i + 1] > 0:
            adv[i] += 1
            adv[i + 1] -= 1
    if max(adv) > 255:
        return None
    diffs = rng.integers(0, 25, len(adv))
    return rec(a, base + bs[0] + off, adv, diffs, e)


def corpus_group(rng, npath=3, nrec=40, length=6000):
    """nrec records cut from npath shared paths (parallel copies a few bases apart in B among them):
    meets, fusions, boxes, shared starts and ends and abpos ties are all common"""
    paths = [(_shared_path(rng, length), int(rng.integers(0, 3)) * 50_000 + 10_000) for _ in range(npath)]
    recs = []
    starts = rng.integers(0, length - 200, 6)
    while len(recs) < nrec:
        path, base = paths[int(rng.integers(0, npath))]
        u = rng.random()
        if recs and u < 0.12:                              # same start, other end / same everything
            r0 = recs[int(rng.integers(0, len(recs)))]
            v = rng.random()
            if v < 0.5:                                    # same ends, other diffs (now and then >= aepos)
                r = dict(r0)
                t = r0["trace"].copy()
                t[0::2] = rng.integers(200, 256, len(t) // 2) if v < 0.15 else rng.integers(0, 25, len(t) // 2)
                r["trace"] = t
                r["diffs"] = int(t[0::2].sum())
                recs.append(r)
                continue
            if v < 0.7 and r0["trace"][1] >= 5:            # same abpos and end, bbpos a little higher
                k = int(rng.integers(1, min(5, int(r0["trace"][1])) + 1))
                t = r0["trace"].copy()
                t[1] -= k
                recs.append(dict(r0, bb=r0["bb"] + k, trace=t))
                continue
        a = int(rng.choice(starts)) if u < 0.3 else int(rng.integers(0, 600 if u < 0.4 else length - 200))
        if rng.random() < 0.2:
            a = (a // TSPACE) * TSPACE
        e = min(length, a + int(rng.integers(20, 2500)))
        if e <= a:
            continue
        off = 0 if rng.random() < 0.6 else int(rng.choice([-12, -11, -10, -9, -5, -3, -1, 1, 2, 4, 9, 10, 11]))
        r = _cut(rng, path, base, a, e, off)
        if r is not None:
            recs.append(r)
    order = rng.permutation(len(recs))
    return [recs[i] for i in order]


def corpus(seed, ngroups=12):
    rng = np.random.default_rng(seed)
    groups = []
    for g in range(ngroups):
        groups.append((int(g % 2), int(g // 4), int((g // 2) % 2), corpus_group(rng, int(rng.integers(1, 4)),
                                                                               int(rng.integers(2, 80)))))
    groups.sort(key=lambda x: (x[0], x[1], x[2]))
    return dict(groups=groups, nA=ngroups // 4 + 1, nB=2, rank1=np.random.default_rng(seed).permutation(ngroups // 4 + 1),
                rank2=np.array([1, 0], np.int32))

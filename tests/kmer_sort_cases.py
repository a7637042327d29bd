"""TEST INFRASTRUCTURE (CPU only): crafted inputs that drive the k-mer table sort (sort128.cu: the partition
passes, kmer_fine_bounds_kernel, kmer_plan_kernel, kmer_bucket_sort_kernel, fgb_kmer_sort_oversized) and the
syncmer scan's emit layout (gix.cu syncmer_body) into their corners, and numpy restatements of the rules that
say which corner an input reaches.

Two kinds of case:
  - a record case is (n, 2) uint64 records in the device layout ([lo, hi], common.cuh) whose 12-base prefixes
    (hi >> 40) lie in [plo, phi), unique, in the order they are handed to fgb_gix_from_records, with the bin
    target the sort runs under (None: the default).  They are built record by record, so bin and sub-bin
    sizes are exact;
  - a genome case is a list of contigs built as a whole table (both strands), a forward-only table or a
    prefix range of a table, for what only the scan route reaches: a first digit (dbits > 0), fine bins
    finer than the sort's bins (fsh < sh), and tiles crowded enough to be staged in rounds.

The kernels' constants are read from the sources, so the restatements follow the kernels."""
import functools
import os
import re

import numpy as np

import oracle_lib as ol
from fastga_b200 import formats

_CSRC = os.path.join(ol.ROOT, "fastga_b200", "csrc")
H100_SMS = 132          # SMs of an H100 SXM; the bucket sort runs two CTAs on each


def _defines(path):
    """the integer #defines of a source file, later ones written in terms of earlier ones"""
    vals = {}
    for m in re.finditer(r"^#define\s+(\w+)\s+([^\n]*)", open(path).read(), re.M):
        expr = m.group(2).split("//")[0].strip()
        for k, v in vals.items():
            expr = re.sub(r"\b%s\b" % k, str(v), expr)
        if expr and re.fullmatch(r"[\d\s()+\-*/<>]+", expr):
            vals[m.group(1)] = int(eval(expr.replace("/", "//")))
    return vals


def _kernel_constants():
    s = _defines(os.path.join(_CSRC, "sort128.cu"))
    g = _defines(os.path.join(_CSRC, "gix.cu"))
    K = {k: s[k] for k in ("BK_CAP", "BK_SPAN", "BK_SUBBITS", "BK_MAXSUB", "SORT_THREADS", "SORT_ITEMS",
                           "SORT_TILE")}
    K.update({k: g[k] for k in ("SC_THREADS", "SC_PPT", "SC_TILE", "SC_STAGE", "SC_ROUNDS", "SC_DBITS")})
    src = open(os.path.join(_CSRC, "sort128.cu")).read()
    m = re.search(r"long long maxbins = (\d+), target = (\d+);", src)
    K["MAXBINS"], K["BIN_TARGET"] = int(m.group(1)), int(m.group(2))
    return K


K = _kernel_constants()
BK_CAP, BK_SPAN, BK_MAXSUB, SORT_TILE = K["BK_CAP"], K["BK_SPAN"], K["BK_MAXSUB"], K["SORT_TILE"]
SC_TILE, SC_STAGE = K["SC_TILE"], K["SC_STAGE"]
TOP = 1 << 24

# ------------------------------------------------------------------------------------------------
#  restatements
# ------------------------------------------------------------------------------------------------


def bin_shift(n, plo, phi, target=None):
    """fgb_kmer_bin_shift: bins of 2^sh prefixes, as many as keep n / bins near the target"""
    maxbins = K["MAXBINS"]
    t = K["BIN_TARGET"] if target is None else max(int(target), 1)
    while maxbins < TOP and n // maxbins > t:
        maxbins <<= 1
    sh = 0
    while ((phi - 1) >> sh) - (plo >> sh) >= maxbins:
        sh += 1
    return sh


def first_digit(nmax, plo, phi, target=None):
    """fgb_kmer_first_digit -> (fsh, dbits): the partition of prefix bits [fsh, 24) is a first digit of dbits
    bits laid out by the scan, then 8-bit Onesweep passes"""
    fsh = bin_shift(nmax, plo, phi, target)
    bits = 24 - fsh
    passes = max(1, (bits - 9 + 7) // 8)
    return fsh, bits - 8 * passes


def partition_passes(b0):
    """Onesweep passes of fgb_kmer_sort_device from record bit b0 = 104 + fsh + dbits"""
    return (128 - b0 + 7) // 8


def plan_groups(bins):
    """the planning kernel's rule on bin starts bins[0..nbins]: windows of BK_SPAN bins, each packed greedily into
    groups (start, count, first bin); bins above BK_CAP records are listed apart as (start, count)"""
    groups, over = [], []
    for w0 in range(0, len(bins) - 1, BK_SPAN):
        gs = gc = gp = 0
        for p in range(w0, min(w0 + BK_SPAN, len(bins) - 1)):
            ln = int(bins[p + 1] - bins[p])
            if ln == 0:
                continue
            if ln > BK_CAP:
                if gc:
                    groups.append((gs, gc, gp))
                    gc = 0
                over.append((int(bins[p]), ln))
                continue
            if gc + ln > BK_CAP:
                groups.append((gs, gc, gp))
                gc = 0
            if gc == 0:
                gs, gp = int(bins[p]), p
            gc += ln
        if gc:
            groups.append((gs, gc, gp))
    return groups, over


def sort_records(recs):
    """the table: records by the whole 128-bit value (hi, then lo)"""
    recs = np.asarray(recs, dtype=np.uint64).reshape(-1, 2)
    return recs[np.lexsort((recs[:, 0], recs[:, 1]))]


def prefix_index(tab):
    """pstart[x] = first entry whose 12-base prefix is >= x, x in [0, 2^24]"""
    pre = tab[:, 1] >> np.uint64(40)
    return np.searchsorted(pre, np.arange(TOP + 1, dtype=np.uint64), side="left").astype(np.uint32)


def record_plan(recs, plo, phi, target=None, sms=H100_SMS):
    """what fgb_kmer_sort_device does with records in any order (dbits = 0: the fine bins are the bins):
    sh, the bins, the plan's groups (in window order) and oversized bins, per group its largest sub-bin, its
    bins with a crowded sub-bin and whether it takes the LSD path, the grid and the CTA of each group when the
    groups are handed out in window order (the kernel's order is the planning kernel's atomic order)"""
    recs = np.asarray(recs, dtype=np.uint64).reshape(-1, 2)
    n = len(recs)
    sh = bin_shift(n, plo, phi, target)
    base = plo >> sh
    nbins = ((phi - 1) >> sh) - base + 1
    tab = sort_records(recs)
    hi = tab[:, 1]
    binof = (hi >> np.uint64(40 + sh)).astype(np.int64) - base
    bins = np.zeros(nbins + 1, dtype=np.int64)
    bins[1:] = np.cumsum(np.bincount(binof, minlength=nbins))
    P = dict(n=n, sh=sh, nbins=nbins, bins=bins, tab=tab, passes=partition_passes(104 + sh),
             grid=min(nbins, 2 * sms), groups=[], over=[])
    if n <= 1:                       # nothing to sort: no pass, no plan
        P["passes"] = 0
        return P
    groups, over = plan_groups(bins)
    sub = (hi >> np.uint64(40 + sh - K["BK_SUBBITS"])).astype(np.int64) & ((1 << K["BK_SUBBITS"]) - 1)
    for gs, gc, gp in groups:
        s = (binof[gs:gs + gc] - gp) * (1 << K["BK_SUBBITS"]) + sub[gs:gs + gc]
        cnt = np.bincount(s, minlength=BK_SPAN << K["BK_SUBBITS"]).reshape(BK_SPAN, -1)
        crowded = [k for k in range(BK_SPAN) if cnt[k].max() > BK_MAXSUB]
        P["groups"].append(dict(start=gs, count=gc, bin=gp, maxsub=int(cnt.max()), crowded=crowded,
                                lsd=bool(crowded)))
    P["over"] = over
    P["ototal"] = sum(c for _, c in over)
    for i, g in enumerate(P["groups"]):
        g["cta"] = i % P["grid"]
    return P


def _input_rank(recs):
    """position in the input of each entry of the sorted table"""
    recs = np.asarray(recs, dtype=np.uint64).reshape(-1, 2)
    return np.lexsort((recs[:, 0], recs[:, 1]))


_LO_CLASSES = (("strand", np.uint64(1 << 47)), ("contig", np.uint64(0x7fff << 32)),
               ("post", np.uint64(0xffffffff)), ("byte0", np.uint64(0xff)))


def record_rows(c, sms=H100_SMS):
    """the rows of ROWS a record case reaches"""
    P = record_plan(c.records, c.plo, c.phi, c.target, sms)
    rows = set()
    n, bins, nbins, sh = P["n"], P["bins"], P["nbins"], P["sh"]
    size = np.diff(bins)
    tiles = {0: "n=0", 1: "n=1", 2: "n=2", SORT_TILE - 1: "n=tile-1", SORT_TILE: "n=tile",
             SORT_TILE + 1: "n=tile+1", 2 * SORT_TILE + 1: "n=2tile+1"}
    if n in tiles:
        rows.add(tiles[n])
    if n <= 1:
        return rows
    rows.add("passes%d" % P["passes"])
    if nbins > 65536:
        rows.add("bins>65536")
    tab = P["tab"]
    hi = tab[:, 1]
    for p in range(P["passes"]):
        b = 104 + sh + 8 * p - 64
        if len(np.unique((hi >> np.uint64(b)) & np.uint64(0xff))) == 1:
            rows.add("one_digit_first" if p == 0 else "one_digit_later")
    # plan
    for s, name in ((1, "bin_1"), (BK_CAP - 1, "bin_cap-1"), (BK_CAP, "bin_cap"), (BK_CAP + 1, "bin_cap+1")):
        if (size == s).any():
            rows.add(name)
    for g in P["groups"]:
        b0, b1 = g["bin"], int(np.searchsorted(bins, g["start"] + g["count"], side="left"))
        if (size[b0:b1] == 0).any():
            rows.add("bin_0")                    # an empty bin inside a group
    for w0 in range(0, nbins, BK_SPAN):
        ws = size[w0:w0 + BK_SPAN]
        small = ws[(ws > 0) & (ws <= BK_CAP)]
        if (ws <= BK_CAP).all() and len(small) >= 2 and small.sum() in (BK_CAP, BK_CAP + 1):
            rows.add("window_cap" if small.sum() == BK_CAP else "window_cap+1")
        for k in range(len(ws)):
            if ws[k] > BK_CAP:
                before, after = (ws[:k] > 0).any(), (ws[k + 1:] > 0).any()
                if k == 0 and after:
                    rows.add("over_slot0")
                if k == 1 and before and after:
                    rows.add("over_slot1")
                if k == 2 and before and after:
                    rows.add("over_flush")
                if k == BK_SPAN - 1 and before:
                    rows.add("over_slot3")
    if nbins % BK_SPAN and size[nbins - nbins % BK_SPAN:].sum() > 0:
        rows.add("nbins%%4=%d" % (nbins % BK_SPAN))
    if nbins == 1:
        rows.add("nbins=1")
    if nbins == 65536 and (size > 0).sum() == 1:
        rows.add("one_bin_of_65536")
    # shares
    if nbins > 1:
        if c.plo % (1 << sh) and size[0] > 0:
            rows.add("plo_unaligned")
        if c.phi % (1 << sh) and size[-1] > 0:
            rows.add("phi_unaligned")
        if c.phi == TOP and c.plo > 0 and size[-1] > 0:
            rows.add("phi_top")
        if size[0] == n:
            rows.add("first_bin_only")
        if size[-1] == n:
            rows.add("last_bin_only")
        if size[0] == 0 and size[-1] == 0:
            rows.add("empty_ends")
    # sub-bins
    for g in P["groups"]:
        if not g["lsd"] and g["maxsub"] in (BK_MAXSUB - 1, BK_MAXSUB):
            rows.add("sub%d" % g["maxsub"])
        if g["lsd"] and g["maxsub"] == BK_MAXSUB + 1:
            rows.add("sub%d" % g["maxsub"])
        if len(g["crowded"]) == BK_SPAN:
            rows.add("crowded_each_bin")
    # ties: adjacent entries equal in hi whose lo differ only in one field, handed in in the other order
    path = np.full(n, "", dtype=object)
    for g in P["groups"]:
        path[g["start"]:g["start"] + g["count"]] = "lsd" if g["lsd"] else "fast"
    rank = _input_rank(c.records)
    eq = np.nonzero((hi[1:] == hi[:-1]) & (rank[1:] < rank[:-1]))[0]
    d = tab[eq + 1, 0] ^ tab[eq, 0]
    for name, mask in _LO_CLASSES:
        for k in eq[(d & ~mask) == 0]:
            if path[k] and path[k] == path[k + 1]:
                rows.add("tie_%s_%s" % (name, path[k]))
    lo16 = np.nonzero((d >> np.uint64(48)) == 0)[0]
    for k in eq[lo16]:
        if path[k] and path[k] == path[k + 1]:
            rows.add("tie_lo16_%s" % path[k])
    # the CTA loop
    ng = len(P["groups"])
    if ng > 3 * P["grid"]:
        rows.add("cta_loop3")
    for cta in range(P["grid"]):
        kinds = [g["lsd"] for g in P["groups"][cta::P["grid"]]]
        if any(a != b and b != c for a, b, c in zip(kinds, kinds[1:], kinds[2:])):
            rows.add("cta_mixed")
            break
    # oversized bins
    over = P["over"]
    if over:
        rows.add({1: "over1", 2: "over2"}.get(len(over), "over3+"))
        if len(over) >= 300:
            rows.add("over300")
        if size[-1] > BK_CAP:
            rows.add("over_last")
        ot = P["ototal"]
        rows.add({SORT_TILE + 1: "ototal=tile+1", 2 * SORT_TILE: "ototal=2tiles"}.get(
            ot, "ototal>2tiles" if ot > 2 * SORT_TILE else "ototal<2tiles"))
        if any(g["lsd"] for g in P["groups"]) and any(not g["lsd"] for g in P["groups"]):
            rows.add("over_lsd_fast")
        if len(over) >= 2:
            first = [int(rank[s:s + l].min()) for s, l in over]
            if all(a < b for a, b in zip(first, first[1:])):
                rows.add("over_asc")
            elif all(a > b for a, b in zip(first, first[1:])):
                rows.add("over_desc")
            else:
                rows.add("over_random")
    return rows


# ------------------------------------------------------------------------------------------------
#  record cases
# ------------------------------------------------------------------------------------------------

class RecordCase:
    def __init__(self, name, records, plo=0, phi=TOP, target=None):
        self.name, self.records, self.plo, self.phi, self.target = name, records, plo, phi, target


class _Records:
    """records put together part by part; every record gets a post of its own unless the part gives them"""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.parts = []
        self.post = 0

    def add(self, prefix, count, hi_low=None, lo_top=None, cont=None, post=None, order="random"):
        """count records of 12-base prefix `prefix` (one or one each); hi_low: hi bits [0,40); lo_top: lo bits
        [48,64); cont: lo bits [32,48) (strand bit 47 on top of the contig rank); post: lo bits [0,32)"""
        rng, u = self.rng, np.uint64

        def field(v, bits):
            if v is None:
                return rng.integers(0, 1 << bits, count, dtype=np.uint64)
            return np.broadcast_to(np.asarray(v, dtype=np.uint64), (count,))

        if post is None:
            post = np.arange(self.post, self.post + count, dtype=np.uint64)
            self.post += count
        hi = (field(prefix, 24) << u(40)) | field(hi_low, 40)
        lo = (field(lo_top, 16) << u(48)) | (field(cont, 16) << u(32)) | field(post, 32)
        r = np.stack([lo, hi], axis=1)
        if order == "random":
            r = r[rng.permutation(count)]
        elif order in ("asc", "desc"):
            r = sort_records(r)[::1 if order == "asc" else -1]
        self.parts.append(r)
        return self

    def in_bin(self, b, count, sh=8, order="random"):
        """count records spread over the prefixes of bin b (bins of 2^sh prefixes)"""
        pre = (b << sh) | self.rng.integers(0, 1 << sh, count, dtype=np.uint64)
        return self.add(pre, count, order=order)

    def sub_bin(self, b, count, sub=1, order="random", **kw):
        """count records of one sub-bin of bin b (sh = 8: the bin's 8 prefix bits below it and hi bits 38-39)"""
        pre = (b << 8) | (sub >> 2)
        low = (np.uint64(sub & 3) << np.uint64(38)) | self.rng.integers(0, 1 << 38, count, dtype=np.uint64)
        return self.add(pre, count, hi_low=kw.pop("hi_low", low), order=order, **kw)

    def in_range(self, lo, hi, count):
        return self.add(self.rng.integers(lo, hi, count, dtype=np.uint64), count)

    def records(self, part_order=None):
        parts = self.parts if part_order is None else [self.parts[i] for i in part_order]
        return np.concatenate(parts) if parts else np.zeros((0, 2), dtype=np.uint64)


def _windows(R, w, sizes):
    for k, s in enumerate(sizes):
        if s:
            R.in_bin(BK_SPAN * w + k, s)


def _tie_sets(R, b, sub, kinds, order="desc"):
    """records equal in hi whose lo differ only in one field, handed in in descending order"""
    rng = R.rng
    for kind in kinds:
        hi_low = (np.uint64(sub & 3) << np.uint64(38)) | rng.integers(0, 1 << 38, dtype=np.uint64)
        top, cont, post = int(rng.integers(1 << 16)), int(rng.integers(1 << 15)), int(rng.integers(1 << 30)) << 1
        pre = (b << 8) | (sub >> 2)
        if kind == "strand":
            R.add(pre, 2, hi_low, top, [cont, cont | 0x8000], post, order)
        elif kind == "contig":
            R.add(pre, 3, hi_low, top, [cont, cont ^ 1, cont ^ 0x4000], post, order)
        elif kind == "post":
            R.add(pre, 3, hi_low, top, cont, [post, post + 1, post + (1 << 31)], order)
        elif kind == "lo16":
            R.add(pre, 2, hi_low, top, [cont, cont ^ 3], [post, post + 5], order)


def _rec_cases():
    C = {}

    def case(name, R, plo=0, phi=TOP, target=None, part_order=None):
        C[name] = (R, plo, phi, target, part_order)

    # --- plan: bins of 0, 1, BK_CAP-1 and BK_CAP records, and no oversized bin (one host wait)
    R = _Records(1)
    _windows(R, 10, [1, 0, 2, 0])
    _windows(R, 20, [BK_CAP - 1])
    _windows(R, 30, [0, 0, BK_CAP])
    _windows(R, 40, [7, 0, 0, 0])
    case("plan_bins_0_1_cap-1_cap", R)
    R = _Records(2)
    _windows(R, 50, [5, BK_CAP + 1, 9])
    case("plan_bin_cap+1", R)
    R = _Records(3)
    _windows(R, 5, [1000, 1000, 1000, BK_CAP - 3000])
    _windows(R, 6, [1000, 1000, 1000, BK_CAP - 2999])
    _windows(R, 7, [BK_CAP // 2, 0, BK_CAP // 2])
    _windows(R, 8, [BK_CAP - 96, 97])
    case("plan_window_sums_cap_cap+1", R)
    R = _Records(4)
    _windows(R, 100, [5000, 7, 9, 0])
    _windows(R, 101, [11, 4500, 13, 0])
    _windows(R, 102, [20, 200, 6000, 50])
    _windows(R, 103, [20, 30, 0, 4200])
    R.sub_bin(800, 40)
    R.in_bin(900, 50)
    case("plan_oversized_slots_0_1_2_3", R, part_order=[9, 3, 7, 0, 12, 5, 1, 11, 2, 10, 4, 6, 8, 13, 14])
    for m, (plo, width) in {1: (3000, 4001), 2: (123456, 4002), 3: ((1 << 23) + 1, 40003)}.items():
        R = _Records(10 + m)
        R.in_range(plo, plo + width, 2000)
        R.add(plo + width - 1, 5)
        R.add(plo, 3)
        case("plan_nbins_mod4_%d" % m, R, plo, plo + width)
    R = _Records(14)
    R.add(777777, 3000)
    case("plan_nbins_1", R, 777777, 777778)
    R = _Records(15)
    R.in_bin(40000, 2000)
    case("plan_one_bin_of_65536", R)
    # --- shares of the prefix space: partial first and last bins, empty ends, the top of the space
    plo, phi = (1 << 20) + 3, (1 << 20) + 300003
    R = _Records(20)
    R.in_range(plo, phi, 3000)
    R.add(plo, 10)
    R.add(phi - 1, 10)
    case("share_unaligned_plo_phi", R, plo, phi)
    R = _Records(21)
    R.in_range(plo, (plo | 7) + 1, 500)
    case("share_first_bin_only", R, plo, phi)
    R = _Records(22)
    R.in_range((phi - 1) & ~7, phi, 500)
    case("share_last_bin_only", R, plo, phi)
    R = _Records(23)
    R.in_range(TOP - 300001, TOP, 3000)
    R.add(TOP - 1, 20)
    case("share_phi_top", R, TOP - 300001, TOP)
    R = _Records(24)
    R.in_range((1 << 22) + 105, (1 << 22) + 499905, 3000)
    case("share_empty_ends", R, (1 << 22) + 5, (1 << 22) + 500005)
    # --- sub-bins of 31, 32 and 33 records; ties in lo
    R = _Records(30)
    R.in_bin(4000, 40)
    R.add((4000 << 8) | 77, 31, hi_low=(1 << 38) | 12345, lo_top=99, cont=5, post=np.arange(31) + (1 << 31),
          order="desc")
    R.in_bin(4100, 40)
    for k in range(8):
        _tie_sets(R, 4100, 700, ["strand"])
    for k in range(5):
        _tie_sets(R, 4100, 700, ["contig"])
    R.sub_bin(4100, 1, 700)
    R.in_bin(4200, 40)
    R.add((4200 << 8) | 3, 33, hi_low=(2 << 38) | 777, lo_top=7, cont=0x8003, post=np.arange(33) + (5 << 28),
          order="desc")
    case("sub_31_32_33", R)
    R = _Records(31)
    R.in_bin(4400, 60)
    _tie_sets(R, 4400, 9, ["strand", "contig", "post", "lo16"] * 3)
    R.in_bin(4500, 60)
    R.sub_bin(4500, 30, 400)
    _tie_sets(R, 4500, 400, ["strand", "contig", "post", "lo16"])
    case("sub_lo_ties_fast_and_lsd", R)
    R = _Records(32)
    for k in range(BK_SPAN):
        R.in_bin(8000 + k, 100)
        R.sub_bin(8000 + k, BK_MAXSUB + 1, 100 + 200 * k)
    case("sub_crowded_in_each_bin", R)
    # --- one CTA runs more than three groups, fast and LSD ones in turn
    R = _Records(33)
    for i in range(1100):
        b = BK_SPAN * (14 * i + 3) + i % BK_SPAN
        if i % 5 in (1, 3):
            R.sub_bin(b, BK_MAXSUB + 2, 555)
        R.in_bin(b, 10 if i % 5 in (1, 3) else 25)
    case("cta_loop_fast_lsd_alternating", R)
    # --- oversized bins
    R = _Records(40)
    R.in_bin(60000, BK_CAP + 4)
    R.in_bin(300, BK_CAP + 1)
    R.sub_bin(500, 35)
    R.in_bin(700, 30)
    case("over_two_descending_lsd_fast", R)
    R = _Records(41)
    R.in_bin(10, BK_CAP + 1)
    R.in_bin(20, BK_CAP + 2)
    R.in_bin(30000, BK_CAP + 3)
    case("over_three_ascending", R)
    R = _Records(42)
    R.in_bin(65535, 2 * SORT_TILE)
    R.in_bin(65533, 100)
    case("over_last_bin_two_tiles", R)
    R = _Records(43)
    for i in range(300):
        R.in_bin(200 * i + 13, BK_CAP + 1 + (7 * i) % 300)
    R.in_range(0, TOP, 2000)
    case("over_300_random", R, part_order=list(np.random.default_rng(43).permutation(301)))
    # --- the partition passes
    for n in (0, 1, 2, SORT_TILE - 1, SORT_TILE, SORT_TILE + 1, 2 * SORT_TILE + 1):
        R = _Records(50 + n % 97)
        R.in_range(0, TOP, n)
        case("part_n%d" % n, R)
    R = _Records(60)
    R.add(np.uint64(0xa5 << 8) | R.rng.integers(0, 256, 5000, dtype=np.uint64)
          | (R.rng.integers(0, 256, 5000, dtype=np.uint64) << np.uint64(16)), 5000)
    case("part_one_first_digit", R)
    R = _Records(61)
    R.in_range(0, TOP, 140000)
    case("part_target1_3passes_131072_bins", R, target=1)
    R = _Records(62)
    R.in_range(0, TOP, 70000)
    case("part_target1_2passes", R, target=1)
    return C


@functools.lru_cache(maxsize=None)
def _rec_case_table():
    return _rec_cases()


RECORD_NAMES = sorted(_rec_case_table())


@functools.lru_cache(maxsize=4)
def record_case(name):
    R, plo, phi, target, order = _rec_case_table()[name]
    return RecordCase(name, R.records(order), plo, phi, target)


# ------------------------------------------------------------------------------------------------
#  genome cases
# ------------------------------------------------------------------------------------------------

def syncmers(seq):
    """sampled positions of a contig (orc_syncmers: closed (12,8)-syncmers, ties included)"""
    seq = np.ascontiguousarray(seq, dtype=np.uint8)
    out = np.zeros(max(len(seq), 1), dtype=np.int64)
    m = ol.orc().orc_syncmers(seq.ctypes.data_as(ol.C.c_void_p), ol.C.c_int64(len(seq)),
                              out.ctypes.data_as(ol.C.c_void_p))
    return out[:m]


def tile_records(seq, fwd_only):
    """records of each 4096-position scan tile of one contig, whole prefix range: a forward entry at every
    sampled j <= L-40, a reverse entry at every sampled j >= 28 (none in a forward-only table)"""
    L = len(seq)
    if L < 12:
        return np.zeros(0, dtype=np.int64)
    pos = syncmers(seq)
    w = (pos <= L - 40).astype(np.int64) + (0 if fwd_only else (pos >= 28))
    return np.bincount(pos // SC_TILE, weights=w, minlength=(L - 12) // SC_TILE + 1).astype(np.int64)


def buck1024(contigs):
    """the sampler histogram: the first five bases of the 12-mer at every sampled position, and of its
    reverse complement, over every contig whatever the range or strand filter of the table"""
    h = np.zeros(1024, dtype=np.int64)
    for s in contigs:
        if len(s) < 12:
            continue
        pos = syncmers(s)
        s = np.asarray(s, dtype=np.int64)
        fb = sum(s[pos + k] << (2 * (4 - k)) for k in range(5))
        rb = sum((3 - s[pos + 11 - k]) << (2 * (4 - k)) for k in range(5))
        h += np.bincount(fb, minlength=1024) + np.bincount(rb, minlength=1024)
    return h


def _crowded(seed, want, fwd_only, tail=4097):
    """a contig of two tiles whose first tile holds exactly `want` records: a run of A inside random bases,
    lengthened until the tile's count lands on want.  The first tile, because a sampled position inside a
    contig gives two records when both strands are kept: only positions near an end give one, so only there can
    a tile's count be odd."""
    def count(seq, r):
        s = seq.copy()
        s[64:64 + r] = 0
        return tile_records(s, fwd_only)[0], s

    for s in range(seed, seed + 40):
        rng = np.random.default_rng(s)
        seq = rng.integers(0, 4, SC_TILE + tail, dtype=np.uint8)
        r0 = 0                            # coarse steps up to near want (the count grows with the run), then one by one
        while r0 + 32 < SC_TILE - 64 and count(seq, r0 + 32)[0] < want - 64:
            r0 += 32
        for r in range(r0, SC_TILE - 64):
            got, out = count(seq, r)
            if got == want:
                return out
            if got > want + 64:
                break
    raise AssertionError("no run length gives a tile of %d records" % want)


class GenomeCase:
    def __init__(self, name, contigs, kind, plo=0, phi=TOP, target=None):
        self.name, self.contigs, self.kind, self.plo, self.phi, self.target = name, contigs, kind, plo, phi, target

    @functools.cached_property
    def genome(self):
        return _genome(self.contigs)

    @property
    def full_range(self):
        return self.kind != "range"


@functools.lru_cache(maxsize=None)
def _contigs(which):
    if which == "stage_both":
        rng = np.random.default_rng(70)
        end = np.concatenate([rng.integers(0, 4, SC_TILE, dtype=np.uint8), np.zeros(2600, dtype=np.uint8)])
        return (_crowded(71, SC_STAGE, False), _crowded(81, SC_STAGE + 1, False, 4098), end,
                rng.integers(0, 4, 20000, dtype=np.uint8))
    if which == "stage_fwd":
        rng = np.random.default_rng(90)
        return (_crowded(91, SC_STAGE, True), _crowded(101, SC_STAGE + 1, True, 4098),
                rng.integers(0, 4, 20011, dtype=np.uint8))
    rng = np.random.default_rng(110)                      # "random": 300 kbp in three contigs
    return tuple(rng.integers(0, 4, n, dtype=np.uint8) for n in (100_000, 100_001, 99_999))


_GENOMES = {}


def _genome(contigs):
    key = id(contigs)
    if key not in _GENOMES:
        _GENOMES[key] = formats.genome_from_arrays(list(contigs))
    return _GENOMES[key]


def _genome_cases():
    C = {"scan_stage_both": ("stage_both", "both", 0, TOP, None),
         "scan_stage_fwd": ("stage_fwd", "forward", 0, TOP, None),
         "scan_digit9_both": ("random", "both", 0, TOP, 5),
         "scan_digit9_fwd": ("random", "forward", 0, TOP, 5),
         "scan_range_fsh3_sh6": ("random", "range", 0, 1 << 22, 1),
         "scan_range_top_unaligned": ("random", "range", (3 << 22) + 77, TOP, 1)}
    for k in range(8):                    # ranges of 2^(16+k) prefixes: fsh = k, first digits of 8, 7, .. 2, 9 bits
        C["scan_range_fsh%d" % k] = ("random", "range", 5 << 20, (5 << 20) + (1 << (16 + k)), None)
    return C


GENOME_NAMES = sorted(_genome_cases())


def genome_case(name):
    which, kind, plo, phi, target = _genome_cases()[name]
    return GenomeCase(name, _contigs(which), kind, plo, phi, target)


def case_table(c, table):
    """the entries of a genome case's table, from the oracle's both-strand table"""
    if c.kind == "forward":
        return table[(table[:, 0] >> np.uint64(47)) & np.uint64(1) == 0]
    if c.kind == "range":
        pre = table[:, 1] >> np.uint64(40)
        return table[(pre >= c.plo) & (pre < c.phi)]
    return table


def scan_layout(c, n):
    """(fsh, dbits, sh) of a genome case's build with n records: the first digit chosen for an upper bound of
    two records per scanned position, the bins for n"""
    npos = sum(len(s) - 11 for s in c.contigs if len(s) >= 12)
    fsh, dbits = first_digit(2 * npos, c.plo, c.phi if c.phi > c.plo else c.plo + 1, c.target)
    return fsh, dbits, bin_shift(n, c.plo, c.phi, c.target)


def tile_of(c, recs, rank):
    """the scan tile of each record: tiles are numbered contig by contig (contigs of 12 bases or more) in
    genome order, 4096 positions each; a reverse entry's post is its position + 12"""
    clen = np.array([len(s) for s in c.contigs], dtype=np.int64)
    ntile = np.where(clen >= 12, (clen - 12) // SC_TILE + 1, 0)
    tbase = np.concatenate([[0], np.cumsum(ntile)])
    perm = np.empty_like(rank)
    perm[rank] = np.arange(len(rank))
    lo = recs[:, 0]
    contig = perm[((lo >> np.uint64(32)) & np.uint64(0x7fff)).astype(np.int64)]
    j = (lo & np.uint64(0xffffffff)).astype(np.int64) - 12 * ((lo >> np.uint64(47)) & np.uint64(1)).astype(np.int64)
    return tbase[contig] + j // SC_TILE, int(tbase[-1])


def scan_key(c, recs, rank, fsh, dbits):
    """where the scan's emit pass puts a record: in runs by the first digit (prefix bits [fsh, fsh+dbits)),
    within a run by tile"""
    tile, ntiles = tile_of(c, recs, rank)
    digit = ((recs[:, 1] >> np.uint64(40 + fsh)) & np.uint64((1 << dbits) - 1)).astype(np.int64)
    return digit * ntiles + tile


def genome_rows(c, table, rank):
    """the rows of ROWS a genome case reaches, given the oracle's both-strand table of its genome"""
    tab = case_table(c, table)
    fsh, dbits, sh = scan_layout(c, len(tab))
    rows = {"width%d" % dbits, "sh-fsh=%s" % (sh - fsh if sh - fsh < 2 else "2+"),
            "scan_passes%d" % ((24 - fsh - dbits) // 8)}
    tile, ntiles = tile_of(c, tab, rank)
    cnt = np.bincount(tile, minlength=ntiles)
    strand = "fwd" if c.kind == "forward" else "both"
    if c.full_range:
        for v, name in ((SC_STAGE, "tile=stage_"), (SC_STAGE + 1, "tile=stage+1_")):
            if (cnt == v).any():
                rows.add(name + strand)
    rows.add("rounds%d" % (K["SC_ROUNDS"] if cnt.max() > SC_STAGE else 1))
    if cnt.max() > SC_STAGE:
        clen = np.array([len(s) for s in c.contigs], dtype=np.int64)
        last = np.cumsum(np.where(clen >= 12, (clen - 12) // SC_TILE + 1, 0)) - 1
        if (cnt[last[clen >= 12]] > SC_STAGE).any():
            rows.add("rounds%d_contig_end" % K["SC_ROUNDS"])
    return rows


# ------------------------------------------------------------------------------------------------
#  the regime table: every row some case must reach
# ------------------------------------------------------------------------------------------------

ROWS = {
    "plan": ["bin_0", "bin_1", "bin_cap-1", "bin_cap", "bin_cap+1", "window_cap", "window_cap+1", "over_slot0",
             "over_slot1", "over_flush", "over_slot3", "nbins%4=1", "nbins%4=2", "nbins%4=3", "nbins=1",
             "one_bin_of_65536"],
    "shares": ["plo_unaligned", "phi_unaligned", "phi_top", "first_bin_only", "last_bin_only", "empty_ends"],
    "sub-bins": ["sub31", "sub32", "sub33", "crowded_each_bin", "tie_strand_fast", "tie_contig_fast",
                 "tie_post_fast", "tie_lo16_fast", "tie_strand_lsd", "tie_contig_lsd", "tie_post_lsd",
                 "tie_lo16_lsd", "tie_byte0_lsd"],
    "CTA loop": ["cta_loop3", "cta_mixed"],
    "oversized": ["over1", "over2", "over3+", "over300", "over_last", "ototal=tile+1", "ototal=2tiles",
                  "ototal>2tiles", "over_asc", "over_desc", "over_random", "over_lsd_fast"],
    "partition": ["n=0", "n=1", "n=2", "n=tile-1", "n=tile", "n=tile+1", "n=2tile+1", "one_digit_first",
                  "passes2", "passes3", "bins>65536"],
    "first digit": ["width%d" % d for d in range(2, K["SC_DBITS"] + 1)] + ["sh-fsh=0", "sh-fsh=1", "sh-fsh=2+",
                                                                            "scan_passes1", "scan_passes2"],
    "tile staging": ["tile=stage_both", "tile=stage+1_both", "tile=stage_fwd", "tile=stage+1_fwd", "rounds1",
                     "rounds4", "rounds4_contig_end"],
}

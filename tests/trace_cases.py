"""Crafted .1aln records for the trace-point seam (fgb_compute_trace_pts, the reference's
Compute_Trace_PTS), shared by the CPU tests (tests/test_trace_cases.py) and the GPU tests
(tests/test_gpu_trace_tiles.py).

Every record comes from a known edit path: a window of A is mutated by a seeded stream of
substitutions, insertions and deletions, the path is cut at every multiple of TSPACE in A, and each
interval becomes a trace pair (differences of the path on it, B advance), the bytes Compress_TraceTo8
leaves.  A strand-C record's path runs against the complement of its B contig, whose coordinates the
record gives, as the .1aln does.  Each case(name) returns a Case; REGIMES states what each must reach.

Also here, independent of the reference: tile_edit_distance (and count_optimal_scripts) by a row DP,
replay of an int script the way ALNtoPAF consumes it, and the rule for which records are bad."""
import functools

import numpy as np

from fastga_b200 import formats, lib

TSPACE = 100


class Case:
    def __init__(self, A, B, rows, traces):
        self.A, self.B = A, B                              # contigs (uint8 0..3)
        self.fields = np.array(rows, dtype=np.int32).reshape(-1, 9)
        self.toff = np.concatenate([[0], np.cumsum([len(t) for t in traces])]).astype(np.int64)[:-1]
        self.pool = (np.concatenate(traces) if traces else np.zeros(0)).astype(np.uint8)

    def alns(self):
        return lib.Alignments(self.fields.copy(), self.toff.copy(), self.pool.copy(), len(self.fields))

    def genomes(self):
        return formats.genome_from_arrays(self.A), formats.genome_from_arrays(self.B)

    def trace(self, i):
        return self.pool[int(self.toff[i]):int(self.toff[i]) + int(self.fields[i, 8])]

    def bseq(self, i):
        """the B sequence record i aligns to: its contig, or the contig's complement on strand C"""
        b = self.B[int(self.fields[i, 2])]
        return (3 - b[::-1]).astype(np.uint8) if self.fields[i, 0] else b

    def aseq(self, i):
        return self.A[int(self.fields[i, 1])]


# ------------------------------------------------------------------------------------------
#  edit paths and the records cut from them
# ------------------------------------------------------------------------------------------

DIAG, INS, DEL = 0, 1, 2          # step of a path: both advance, B base inserted, A base deleted


def random_steps(rng, m, ins=0.0, dele=0.0, lens=(1, 3)):
    """a path over m A bases: at each A base an insertion (before it) or a deletion run starts with the
    given rates, lengths uniform in lens"""
    steps, i = [], 0
    while i < m:
        r = rng.random()
        if r < ins:
            steps += [INS] * int(rng.integers(lens[0], lens[1] + 1))
        elif r < ins + dele:
            n = min(int(rng.integers(lens[0], lens[1] + 1)), m - i)
            steps += [DEL] * n
            i += n
            continue
        steps.append(DIAG)
        i += 1
    return np.array(steps, dtype=np.int8)


def apply_steps(rng, a, steps, sub=0.0):
    """the B window that `steps` aligns to window a: diagonal bases copied (substituted at rate sub),
    inserted bases random"""
    out, i = [], 0
    for s in steps:
        if s == DIAG:
            c = int(a[i])
            if sub and rng.random() < sub:
                c = (c + int(rng.integers(1, 4))) & 3
            out.append(c)
            i += 1
        elif s == INS:
            out.append(int(rng.integers(0, 4)))
        else:
            i += 1
    assert i == len(a)
    return np.array(out, dtype=np.uint8)


def cut_trace(a, b, ab, bb, steps):
    """trace pairs of the path `steps` from (ab, bb) through contig a and B strand b: cut where the path
    first reaches each multiple of TSPACE strictly inside (ab, ae); per interval (its differences on
    the path, its B advance)"""
    st = np.asarray(steps)
    pa = ab + np.concatenate([[0], np.cumsum(st != INS)])
    pb = bb + np.concatenate([[0], np.cumsum(st != DEL)])
    cost = np.ones(len(st), dtype=np.int64)
    dg = np.flatnonzero(st == DIAG)
    cost[dg] = a[pa[dg]] != b[pb[dg]]
    ae = int(pa[-1])
    xs = np.arange((ab // TSPACE + 1) * TSPACE, ae, TSPACE)
    bounds = np.concatenate([[0], np.searchsorted(pa, xs, "left"), [len(st)]])
    csum = np.concatenate([[0], np.cumsum(cost)])
    d = csum[bounds[1:]] - csum[bounds[:-1]]
    adv = pb[bounds[1:]] - pb[bounds[:-1]]
    assert (adv <= 255).all() and (d <= 255).all()
    tr = np.empty(2 * len(d), dtype=np.uint8)
    tr[0::2], tr[1::2] = d, adv
    return tr, int(pa[-1]), int(pb[-1]), int(cost.sum())


class Builder:
    """records on contig pairs of their own: record k aligns A contig k with B contig k"""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.A, self.B, self.rows, self.traces = [], [], [], []

    def path(self, window, steps, sub=0.0, comp=0, pre=(0, 0), post=(0, 0), a=None):
        """one record: A contig = pre[0] random bases + A window + post[0]; the aligned B strand = pre[1]
        + the mutated window + post[1]; returns the record's index"""
        rng = self.rng
        wa = rng.integers(0, 4, window, dtype=np.uint8) if a is None else np.asarray(a, dtype=np.uint8)
        wb = apply_steps(rng, wa, steps, sub)
        A = np.concatenate([rng.integers(0, 4, pre[0], dtype=np.uint8), wa, rng.integers(0, 4, post[0], dtype=np.uint8)])
        b = np.concatenate([rng.integers(0, 4, pre[1], dtype=np.uint8), wb, rng.integers(0, 4, post[1], dtype=np.uint8)])
        tr, ae, be, diffs = cut_trace(A, b, pre[0], pre[1], steps)
        return self.add(A, b, comp, pre[0], pre[1], ae, be, diffs, tr)

    def add(self, A, b, comp, ab, bb, ae, be, diffs, tr):
        k = len(self.rows)
        self.A.append(A)
        self.B.append((3 - b[::-1]).astype(np.uint8) if comp else b)
        self.rows.append([comp, k, k, ab, bb, ae, be, diffs, len(tr)])
        self.traces.append(np.asarray(tr, dtype=np.uint8))
        return k

    def case(self):
        return Case(self.A, self.B, self.rows, self.traces)


def _div_steps(rng, m, rate):
    """(steps, substitution rate) of a path at divergence `rate`: substitutions at `rate`, and insertion
    and deletion runs of 1-4 bases each starting at rate / 5 per base"""
    return random_steps(rng, m, ins=rate / 5, dele=rate / 5, lens=(1, 4)), rate


def divergence():
    bd = Builder(71)
    for rate in (0.0, 0.01, 0.10, 0.25, 0.35):
        for comp in (0, 1):
            m = int(bd.rng.integers(900, 1400))
            steps, sub = _div_steps(bd.rng, m, rate)
            bd.path(m, steps, sub, comp, pre=(int(bd.rng.integers(0, 300)), int(bd.rng.integers(0, 300))),
                    post=(50, 50))
    return bd.case()


def tile_shapes():
    bd = Builder(72)
    r = bd.rng
    for comp in (0, 1):
        st, sub = _div_steps(r, 700, 0.08)
        bd.path(700, st, sub, comp, pre=(300, 120), post=(40, 40))          # start on a trace point
        st, sub = _div_steps(r, 701, 0.08)
        bd.path(701, st, sub, comp, pre=(199, 77), post=(40, 40))           # start one base before one
        st, sub = _div_steps(r, 640, 0.08)
        bd.path(640, st, sub, comp, pre=(160, 10), post=(40, 40))           # end on a trace point
        st, sub = _div_steps(r, 541, 0.08)
        bd.path(541, st, sub, comp, pre=(260, 10), post=(40, 40))           # end one base past one
        st, sub = _div_steps(r, 60, 0.1)
        bd.path(60, st, sub, comp, pre=(120, 33), post=(40, 40))            # inside one interval
        bd.path(1, np.array([DIAG], np.int8), 0.0, comp, pre=(57, 9), post=(40, 40))    # one base, match
        bd.path(1, np.array([DIAG], np.int8), 1.0, comp, pre=(99, 9), post=(40, 40))    # one base, mismatch
        # a whole interval deleted (B advance 0, M - N = 100) and 155 bases inserted in another
        # (B advance 255, N - M = 155)
        st = np.concatenate([np.zeros(150, np.int8), np.full(100, DEL, np.int8), np.zeros(80, np.int8),
                             np.full(155, INS, np.int8), np.zeros(170, np.int8)])
        bd.path(500, st, 0.03, comp, pre=(50, 50), post=(40, 40))
        # the same shapes with indels in the neighbouring tiles too
        st = np.concatenate([random_steps(r, 250, 0.02, 0.02), np.full(100, DEL, np.int8),
                             random_steps(r, 30, 0.02, 0.02), np.full(155, INS, np.int8), random_steps(r, 170, 0.02, 0.02)])
        bd.path(550, st, 0.05, comp, pre=(0, 31), post=(40, 40))
    return bd.case()


def contig_ends():
    bd = Builder(73)
    r = bd.rng
    for comp in (0, 1):
        for m in (1234, 73, 500, 100, 99):
            st, sub = _div_steps(r, m, 0.06)
            bd.path(m, st, sub, comp)                                       # ab = bb = 0, ae = alen, be = blen
        st, sub = _div_steps(r, 800, 0.06)
        bd.path(800, st, sub, comp, pre=(0, 0), post=(0, 37))               # both starts, A end
        bd.path(800, st, sub, comp, pre=(37, 0), post=(0, 0))               # B start, both ends
    return bd.case()


def _tie_window(rng, m):
    """homopolymer runs and 2-3-base tandem repeats"""
    parts, n = [], 0
    while n < m:
        if rng.random() < 0.5:
            p = np.full(int(rng.integers(4, 14)), int(rng.integers(0, 4)), np.uint8)
        else:
            unit = rng.integers(0, 4, int(rng.integers(2, 4)), dtype=np.uint8)
            p = np.tile(unit, int(rng.integers(3, 7)))
        parts.append(p)
        n += len(p)
    return np.concatenate(parts)[:m]


def ties():
    bd = Builder(74)
    r = bd.rng
    for comp in (0, 1):
        for rate in (0.03, 0.08):
            m = 900
            a = _tie_window(r, m)
            st = random_steps(r, m, ins=rate, dele=rate, lens=(1, 3))
            bd.path(m, st, rate / 3, comp, pre=(41, 13), post=(40, 40), a=a)
    return bd.case()


def _diag_subs(bd, m, sub, comp, pre):
    return bd.path(m, np.zeros(m, np.int8), sub, comp, pre=pre, post=(30, 30))


@functools.lru_cache(maxsize=None)
def _recorded_base():
    """the paths recorded_diffs rewrites: a mix of divergences and shapes on both strands"""
    bd = Builder(75)
    r = bd.rng
    for comp in (0, 1):
        _diag_subs(bd, 600, 0.10, comp, (0, 0))
        for rate in (0.05, 0.15, 0.30):
            st, sub = _div_steps(r, 1000, rate)
            bd.path(1000, st, sub, comp, pre=(37, 80), post=(30, 30))
        st = random_steps(r, 800, 0.05, 0.05, (1, 3))
        bd.path(800, st, 0.02, comp, pre=(0, 5), post=(30, 30), a=_tie_window(r, 800))
    return bd.case()


def _with_diffs(base, fn):
    """base with every record's diff bytes replaced by fn(k, tile eds, tile |M-N|) (None: dropped)"""
    eds = tile_eds(base)
    rows, traces, A, B = [], [], [], []
    for k in range(len(base.fields)):
        tr = base.trace(k).copy()
        new = fn(k, np.array(eds[k]), np.array([abs(t[1] - t[3]) for t in tiles(base.fields[k], tr)]))
        if new is None:
            continue
        tr[0::2] = np.asarray(new)
        f = base.fields[k].copy()
        f[1] = f[2] = len(rows)
        f[7] = int(np.asarray(new).sum())
        rows.append(f)
        traces.append(tr)
        A.append(base.A[k])
        B.append(base.B[k])
    return Case(A, B, rows, traces)


def _even(x):
    return int(x) + (int(x) & 1)


def recorded_diffs():
    base = _recorded_base()
    rng = np.random.default_rng(76)
    parts = []
    # (a) the exact tile optimum
    parts.append(_with_diffs(base, lambda k, ed, dl: ed))
    # (b) the optimum plus slack, up to 255
    parts.append(_with_diffs(base, lambda k, ed, dl: np.minimum(ed + rng.integers(0, 200, len(ed)), 255)))
    parts.append(_with_diffs(base, lambda k, ed, dl: np.full(len(ed), 255)))

    # (c) some tiles understated, the record's even-rounded max still covers every tile
    def under_ok(k, ed, dl):
        d = ed.copy()
        if len(d) < 2:
            return None
        low = np.argsort(ed)[:max(1, len(ed) // 2)]
        d[low] = np.where(rng.random(len(low)) < 0.5, 0, ed[low] // 2)
        if d.max() > 0 and d.max() % 2 == 0:
            d[int(np.argmax(d))] -= 1                   # odd max: only the even rounding covers the top tile
        if (ed - dl > _even(d.max())).any():
            return None
        return d
    parts.append(_with_diffs(base, under_ok))

    # (d) every tile understated so that some tile's wave count passes the max
    def under_bad(k, ed, dl):
        d = ed // 3
        return d if (ed - dl > _even(d.max())).any() else None
    parts.append(_with_diffs(base, under_bad))
    # (e) tlen = 0: exact, indels only, with mismatches
    bd = Builder(77)
    for comp in (0, 1):
        for m, sub, st in ((1500, 0.0, None), (60, 0.0, None), (80, 0.0, "del"), (80, 0.0, "ins"),
                           (600, 0.1, None), (60, 0.05, None)):
            steps = np.zeros(m, np.int8)
            if st == "del":
                steps[20:25] = DEL
            elif st == "ins":
                steps = np.concatenate([steps[:30], np.full(4, INS, np.int8), steps[30:]])
            k = bd.path(m, steps, sub, comp, pre=(213, 7), post=(20, 20))
            if sub:
                bd.traces[k][0::2] = np.minimum(bd.traces[k][0::2], 255)
            bd.rows[k][8] = 0
            bd.traces[k] = bd.traces[k][:0]
    parts.append(bd.case())
    # 600 bp of 10 % substitutions with the byte of every third tile zeroed: covered by the others
    ex = _with_diffs(base, lambda k, ed, dl: None if k != 0 else np.where(np.arange(len(ed)) % 3 == 1, 0, ed))
    parts.append(ex)
    return _concat(parts)


def _concat(cases):
    A, B, rows, traces = [], [], [], []
    for c in cases:
        for k in range(len(c.fields)):
            f = c.fields[k].copy()
            f[1] = f[2] = len(rows)
            rows.append(f)
            traces.append(c.trace(k))
            A.append(c.A[k])
            B.append(c.B[k])
    return Case(A, B, rows, traces)


WIDE_TILES = 12_600                 # per strand: about 25 000 tiles in all


def wide_slab():
    """exact-match tiles whose diff bytes say 250: a slab of about 194 KB each, past 2^32 bytes in all"""
    bd = Builder(78)
    for comp in (0, 1):
        m = WIDE_TILES * TSPACE
        k = _diag_subs(bd, m, 0.0, comp, (0, 0))
        bd.traces[k][0::2] = 250
        bd.rows[k][7] = 250 * WIDE_TILES
    return bd.case()


def self_records():
    """the SELF-mode records of the `dup` genome of test_oracle_pin (the path's records, which
    tests/test_gpu_self.py pins to the oracle's): A and B are the same genome"""
    import oracle_lib as ol
    from test_oracle_pin import _self_genomes
    contigs = _self_genomes()["dup"]
    al = ol.oracle_pipeline_self(formats.genome_from_arrays(contigs))["alns"]
    c = Case(contigs, contigs, al.fields, [al.trace(i) for i in range(len(al))])
    return c


CASES = {"divergence": divergence, "tile_shapes": tile_shapes, "contig_ends": contig_ends, "ties": ties,
         "recorded_diffs": recorded_diffs, "wide_slab": wide_slab, "self_records": self_records}

#  what each case must reach (tests/test_trace_cases.py checks it):
#    strands: both strands present; max_diff_over: some tile's recorded diffs above it; bad / good:
#    some records the rule below rejects / accepts; shapes: tile shapes (see tile_shape_flags); ends:
#    records touching both ends of both contigs; short_contig / hundred_contig: contigs < 100 bp and of
#    a multiple of 100; ties: a tile with more than one optimal script; understated: a record the
#    reference accepts although a tile's byte is below its optimum; tlen0: tlen = 0 records, accepted
#    and rejected; slab_over: the first launch's slabs pass 2^32 bytes
REGIMES = {"divergence": dict(strands=True, max_diff_over=60, good=True),
           "tile_shapes": dict(strands=True, shapes=("start_on", "start_99", "end_on", "end_past1", "tlen2",
                                                     "one_base", "badv0", "badv255", "del_ge100", "ins_ge100"),
                               good=True),
           "contig_ends": dict(strands=True, ends=True, short_contig=True, hundred_contig=True, good=True),
           "ties": dict(strands=True, ties=True, good=True),
           "recorded_diffs": dict(strands=True, bad=True, good=True, understated=True, tlen0=True, slack255=True),
           "wide_slab": dict(strands=True, slab_over=1 << 32, good=True),
           "self_records": dict(strands=True, good=True)}


@functools.lru_cache(maxsize=None)
def case(name):
    return CASES[name]()


def reference_run(name):
    """the reference's script key (or "fail") of every record of case `name` (oracle_lib.reference)"""
    import oracle_lib as ol
    c = case(name)
    gA, gB = c.genomes()
    return ol.reference("trace_tiles/" + name, ol.digest(c.A, c.B, c.fields, c.pool),
                        lambda: ol.ref_trace_pts(c.alns(), gA, gB))


# ------------------------------------------------------------------------------------------
#  an independent restatement of what a record means
# ------------------------------------------------------------------------------------------

def tiles(f, tr):
    """the tiles of record f (its 9 fields) with trace bytes tr: (a0, m, b0, n, recorded diffs)"""
    ab, bb, ae, be, tlen = int(f[3]), int(f[4]), int(f[5]), int(f[6]), int(f[8])
    nt = tlen // 2 if tlen >= 2 else 1
    out, a, b = [], ab, bb
    for t in range(nt):
        last = t == nt - 1
        e = ae if last else (ab // TSPACE) * TSPACE + (t + 1) * TSPACE
        eb = be if last else b + int(tr[2 * t + 1])
        out.append((a, e - a, b, eb - b, int(tr[2 * t]) if tlen >= 2 else 0))
        a, b = e, eb
    return out


def record_dmax(f, tr):
    """the wave limit of every tile of the record: its largest diff byte rounded up to even, 0 when
    tlen < 2"""
    if int(f[8]) < 2:
        return 0
    return _even(int(np.asarray(tr[0::2]).max()))


def tile_edit_distance(a, b):
    """unit-cost edit distance of a and b: a row DP over a, the moves along b by a running minimum"""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    if len(a) == len(b) and (a == b).all():
        return 0
    j = np.arange(len(b) + 1)
    row = j.copy()
    for i in range(len(a)):
        diag = row[:-1] + (b != a[i])
        nxt = np.empty_like(row)
        nxt[0] = i + 1
        nxt[1:] = np.minimum(diag, row[1:] + 1)
        row = np.minimum.accumulate(nxt - j) + j
    return int(row[-1])


def count_optimal_scripts(a, b):
    """(edit distance, number of distinct optimal alignments) of a and b"""
    m, n = len(a), len(b)
    cost = [[0] * (n + 1) for _ in range(m + 1)]
    cnt = [[0] * (n + 1) for _ in range(m + 1)]
    for i in range(m + 1):
        for j in range(n + 1):
            if i == 0 and j == 0:
                cnt[0][0] = 1
                continue
            best, ways = 1 << 30, 0
            for c, w in (((cost[i - 1][j - 1] + (a[i - 1] != b[j - 1]), cnt[i - 1][j - 1]) if i and j else (1 << 30, 0)),
                         ((cost[i - 1][j] + 1, cnt[i - 1][j]) if i else (1 << 30, 0)),
                         ((cost[i][j - 1] + 1, cnt[i][j - 1]) if j else (1 << 30, 0))):
                if c < best:
                    best, ways = c, w
                elif c == best:
                    ways += w
            cost[i][j], cnt[i][j] = best, ways
    return cost[m][n], cnt[m][n]


def _tile_eds(c, k):
    a, b = c.aseq(k), c.bseq(k)
    return [tile_edit_distance(a[a0:a0 + m], b[b0:b0 + n]) for a0, m, b0, n, _ in tiles(c.fields[k], c.trace(k))]


_eds_cache = {}


def tile_eds(c):
    """per record, the edit distance of each of its tiles"""
    if id(c) not in _eds_cache:
        _eds_cache[id(c)] = (c, [_tile_eds(c, k) for k in range(len(c.fields))])
    return _eds_cache[id(c)][1]


def expect_bad(c):
    """per record, whether the reference rejects it: some tile needs more waves (edit distance - |M-N|)
    than the record's wave limit"""
    eds = tile_eds(c)
    out = []
    for k in range(len(c.fields)):
        dm = record_dmax(c.fields[k], c.trace(k))
        out.append(any(e - abs(m - n) > dm for e, (a0, m, b0, n, _) in zip(eds[k], tiles(c.fields[k], c.trace(k)))))
    return np.array(out, dtype=bool)


def replay(script, f, a, b):
    """Walk an int script the way ALNtoPAF.c:351-420 consumes it (p < 0: B has an extra base before A
    position -p; p > 0: A has an extra base before B position p, both 1-based) from the record's start
    (f: its 9 fields) over A contig a and B strand b.  Asserts every diagonal run is non-negative, the
    walk ends exactly at (aepos, bepos) and passes through every trace point (so every entry lies
    inside its own tile's box).  Returns (mismatches plus indels of the walk, the A and B positions it
    visits)."""
    ab, bb, ae, be = int(f[3]), int(f[4]), int(f[5]), int(f[6])
    s = np.asarray(script, dtype=np.int64)
    k, h = ab, bb                                  # next A and B base, 0-based
    runs, kinds = [], []
    for p in s:
        if p < 0:
            run = -p - 1 - k
            kinds.append(INS)
        else:
            run = p - 1 - h
            kinds.append(DEL)
        assert run >= 0, ("script entry behind the walk", int(p), k, h)
        runs.append(run)
        k += run + (kinds[-1] == DEL)
        h += run + (kinds[-1] == INS)
    assert ae - k == be - h and ae - k >= 0, ("the walk does not end at the record's end", k, h, ae, be)
    runs.append(ae - k)
    kinds.append(-1)
    seq = np.empty(2 * len(runs), dtype=np.int64)
    cnt = np.empty(2 * len(runs), dtype=np.int64)
    seq[0::2], seq[1::2] = DIAG, kinds
    cnt[0::2], cnt[1::2] = runs, 1
    st = np.repeat(seq, cnt)[:-1]
    pa = ab + np.concatenate([[0], np.cumsum(st != INS)])
    pb = bb + np.concatenate([[0], np.cumsum(st != DEL)])
    dg = np.flatnonzero(st == DIAG)
    cost = int((a[pa[dg]] != b[pb[dg]]).sum()) + int((st != DIAG).sum())
    return cost, pa, pb


def check_script(script, diffs, f, tr, a, b, eds):
    """what any correct Compute_Trace_PTS result satisfies: the replayed cost equals diffs, diffs equals
    the sum of the tile edit distances, the walk passes through every trace point"""
    cost, pa, pb = replay(script, f, a, b)
    assert cost == diffs, (cost, diffs)
    assert diffs == sum(eds), (diffs, sum(eds))
    tl = tiles(f, tr)
    key = pa * (1 << 32) + pb
    pts = np.array([(a0 * (1 << 32) + b0) for a0, _, b0, _, _ in tl[1:]], dtype=np.int64)
    assert np.isin(pts, key).all(), "the walk misses a trace point"

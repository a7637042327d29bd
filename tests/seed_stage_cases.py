"""Crafted seed records of the seed stage: the band segments (seg_scan_kernel, 2048-seed tiles and a decoupled
look-back), the prefilter (seed bound, PREF_LONG, serial_has_chain), the long-triple launch order and the
unsorted order past 2^20 long triples (extend.cu, extend_triples).  Each case is seed records in the form the
merge emits -- SEED_DT rows packed by oracle_lib.seed_records -- with its layout, its chain parameters, the
genomes the extension runs on when it has them, and the edges it claims to hit, each a predicate over the
numpy restatement of its triples and the oracle's chain scan (facts()).  Shared by the CPU pins
(test_seed_stage_cases.py) and the GPU test (test_gpu_seed_stage_cases.py)."""
import numpy as np

import oracle_lib as ol
import wave_cases as wc
from fastga_b200 import formats

PREF_LONG = 64                 # a triple with more seeds is long
SEG_TILE = 2048                # seeds a tile of the segment pass
LONG_SORT_CAP = 1 << 20        # the most long triples put in launch order by a sort
STRAY = 2100                   # anti-diagonals between stray seeds: more than chain_break + 80
CB, CM = 2000, 170             # chain_break, chain_min unless a case says otherwise

# the layout of the small cases: 4 contigs a side, amx + bmx = 2^20 - 1, so the top band is 2^14 - 1 (all
# ones in its 14 bits); the band of diagonal 0 (d = diag - bmx) is MID, and anti-diagonals from A0 up keep
# every post of a band within +-300 of MID inside the contigs
AMX, BMX = 1 << 19, (1 << 19) - 1
LAYOUT = (20, 14, 2, 2, AMX, BMX)
MID = BMX >> 6
A0 = 600_000


def seed_rows(layout, comp, ic, jc, band, anti, plen=40, dlow=0):
    """SEED_DT rows whose records hold these fields (arrays or scalars): the posts solved from the
    diagonal band*64 + dlow and the anti-diagonal (orc_seed_records); the low bit of dlow is set to the
    parity the posts need"""
    amx, bmx = layout[4], layout[5]
    anti = np.atleast_1d(np.asarray(anti, np.int64))
    f = [np.broadcast_to(np.asarray(v, np.int64), anti.shape) for v in (comp, ic, jc, band, plen, dlow)]
    comp, ic, jc, band, plen, dlow = f
    dlow = (dlow & ~1) | ((anti + bmx) & 1)
    diag = band * 64 + dlow
    ip = np.where(comp == 0, anti + diag - bmx, 2 * amx + bmx - diag - anti) // 2
    jp = np.where(comp == 0, anti - diag + bmx, bmx - diag + anti) // 2
    assert (ip >= 0).all() and (jp >= 0).all() and (ip < 1 << 32).all() and (jp < 1 << 32).all()
    r = np.zeros(len(anti), dtype=ol.SEED_DT)
    r["plen"], r["comp"], r["icont"], r["jcont"], r["ipost"], r["jpost"] = plen, comp, ic, jc, ip, jp
    return r


def dense(k, a=A0, step=3):
    """k seeds 3 anti-diagonals apart: with 40-base seeds one chain that qualifies once k >= 31"""
    return a + step * np.arange(k)


def stray(k, a=A0):
    """k seeds STRAY anti-diagonals apart: each its own chain of coverage 80"""
    return a + STRAY * np.arange(k)


def decode(recs, layout):
    """per record (comp, ic, jc, band, anti, lcp); keys of at most 64 bits"""
    anti_b, band_b, jc_b, ic_b = layout[:4]
    assert not recs[:, 1].any()
    lo = recs[:, 0].astype(np.uint64)

    def f(pos, n):
        return ((lo >> np.uint64(pos)) & np.uint64((1 << n) - 1)).astype(np.int64)
    p = 12 + anti_b
    return dict(comp=f(p + band_b + jc_b + ic_b, 1), ic=f(p + band_b + jc_b, ic_b), jc=f(p + band_b, jc_b),
                band=f(p, band_b), anti=f(12, anti_b), lcp=f(0, 6))


def triples(recs, layout, chain_min):
    """the band segments of sorted records and, per segment, the end of its triple, isnew, whether it is
    scanned and whether the prefilter's seed bound keeps it (FastGA.c's triple walk, restated); keys of at
    most 64 bits"""
    anti_b, band_b = layout[:2]
    assert not recs[:, 1].any()
    lo = recs[:, 0]
    n = len(lo)
    if n == 0:
        z = np.zeros(0, np.int64)
        return dict(seg=z, e=z, isnew=z.astype(bool), above=z.astype(bool), scanned=z.astype(bool),
                    kept=z.astype(bool), grp=z, band=z)
    p_band = 12 + anti_b
    up = lo >> np.uint64(p_band)
    seg = np.concatenate([[0], np.nonzero(up[1:] != up[:-1])[0] + 1]).astype(np.int64)
    ends = np.append(seg[1:], n).astype(np.int64)
    d = decode(recs[seg], layout)
    g = (d["comp"] << 40) | (d["ic"] << 20) | d["jc"]
    b = d["band"]
    above = np.append((g[1:] == g[:-1]) & (b[1:] == b[:-1] + 1), False)
    isnew = ~np.append(False, above[:-1])
    e = ends.copy()
    e[above] = ends[np.nonzero(above)[0] + 1]
    scanned = isnew | above
    kept = scanned & (e - seg >= (chain_min + 79) // 80)
    return dict(seg=seg, e=e, isnew=isnew, above=above, scanned=scanned, kept=kept, grp=g, band=b)


class Facts:
    """the numpy triples and the oracle's chain scan of a case"""

    def __init__(self, c):
        self.n = len(c.recs)
        T = triples(c.recs, c.layout, c.chain_min)
        self.__dict__.update(T)
        self.size = self.e - self.seg
        self.long = self.kept & (self.size > PREF_LONG)
        self.otr, self.oh = ol.chains(c.recs, c.layout, c.chain_break, c.chain_min)
        self.has_chain = {int(b) for b in self.otr["b"][self.otr["nh"] > 0]}
        self.nh = dict(zip(self.otr["b"].tolist(), self.otr["nh"].tolist()))
        self.lj = np.nonzero(self.long)[0]
        self.lj = self.lj[np.lexsort((self.lj, -self.size[self.lj]))]       # launch order
        self.nlong = len(self.lj)
        self.lcap = self.n // 32 + 2
        sj = np.nonzero(self.kept & (self.size <= PREF_LONG))[0]
        self.short_work = {int(self.seg[j]) for j in sj if int(self.seg[j]) in self.has_chain}
        self.sbits, self.jbits = int(self.n).bit_length(), int(len(self.seg)).bit_length()

    def at(self, comp, ic, jc, band):
        """index of the segment of (strand, contig pair, band)"""
        q = np.nonzero((self.grp == ((comp << 40) | (ic << 20) | jc)) & (self.band == band))[0]
        assert len(q) == 1, (comp, ic, jc, band)
        return int(q[0])

    def chain(self, comp, ic, jc, band):
        """chains the oracle finds in the triple whose lower band this is (None: not scanned)"""
        return self.nh.get(int(self.seg[self.at(comp, ic, jc, band)]))


class Case:
    def __init__(self, name, family, layout=LAYOUT, chain_break=CB, chain_min=CM):
        self.name, self.family, self.layout = name, family, layout
        self.chain_break, self.chain_min = chain_break, chain_min
        self.rows, self.edges, self.genomes = [], [], None
        self._facts = None

    def add(self, comp, ic, jc, band, anti, plen=40, dlow=0):
        self.rows.append(seed_rows(self.layout, comp, ic, jc, band, anti, plen, dlow))

    def edge(self, what, pred):
        """an edge the case claims to hit: a predicate over its Facts"""
        self.edges.append((what, pred))

    def finish(self, genomes=False):
        rows = np.concatenate(self.rows) if self.rows else np.zeros(0, ol.SEED_DT)
        packed = ol.seed_records(rows, self.layout, sort=False)
        self.recs = packed[np.argsort(packed[:, 0], kind="stable")] if len(packed) else packed
        if genomes is True:
            self.genomes = small_genomes()
        elif genomes:
            self.genomes = genomes
        self.nrows = len(rows)
        self.posts_ok = _posts_inside(rows, self.genomes) if self.genomes is not None else None
        del self.rows
        return self

    @property
    def facts(self):
        if self._facts is None:
            self._facts = Facts(self)
        return self._facts


def _posts_inside(rows, genomes):
    """every seed lies inside its contig pair (ranks by decreasing length)"""
    A, B = genomes
    la = np.sort(np.array([len(a) for a in A]))[::-1]
    lb = np.sort(np.array([len(b) for b in B]))[::-1]
    alen, blen = la[rows["icont"]], lb[rows["jcont"]]
    p = rows["plen"].astype(np.int64)
    ip, jp = rows["ipost"].astype(np.int64), rows["jpost"].astype(np.int64)
    jin = np.where(rows["comp"] == 0, jp + p <= blen, (jp >= p) & (jp <= blen))
    return bool(((ip + p <= alen) & jin).all())


_small = None


def small_genomes():
    """random contigs of lengths AMX, AMX-2, .. and BMX, BMX-2, ..: the layout LAYOUT"""
    global _small
    if _small is None:
        rng = np.random.default_rng(77)
        _small = ([rng.integers(0, 4, AMX - 2 * c, dtype=np.uint8) for c in range(4)],
                  [rng.integers(0, 4, BMX - 2 * c, dtype=np.uint8) for c in range(4)])
    return _small


# ------------------------------------------------------------------------------------------------
#  segment-scan tiles
# ------------------------------------------------------------------------------------------------

def _tile_case(n, pattern):
    """n seeds in dense segments on one contig pair, the bands consecutive but for a gap after every
    third segment; segments start at tile offsets 0, 1 and 2047 of every tile ("edges") or every 1500
    seeds, across tile edges ("cross")"""
    c = Case("tiles_%d_%s" % (n, pattern), "tiles")
    if pattern == "edges":
        starts = sorted({t * SEG_TILE + o for t in range((n + SEG_TILE - 1) // SEG_TILE) for o in (0, 1, SEG_TILE - 1)
                         if t * SEG_TILE + o < n})
    else:
        starts = list(range(0, n, 1500))
    sizes = np.diff(starts + [n])
    for i, k in enumerate(sizes):
        c.add(0, 0, 0, MID - 150 + i + i // 3, dense(int(k)))
    c.edge("n = %d" % n, lambda F, n=n: F.n == n)
    c.edge("segments start where they were put", lambda F, s=starts: F.seg.tolist() == s)
    if pattern == "edges":
        for o in (0, 1, SEG_TILE - 1):
            if o < n:
                c.edge("a segment starts at tile offset %d of every tile that reaches it" % o,
                       lambda F, o=o: all(t * SEG_TILE + o in set(F.seg.tolist())
                                          for t in range((F.n - o + SEG_TILE - 1) // SEG_TILE)))
    else:
        c.edge("segments cross tile edges", lambda F: any(s % SEG_TILE + sz > SEG_TILE for s, sz in
                                                           zip(F.seg.tolist(), np.diff(F.seg.tolist() + [F.n]))))
    c.edge("the last tile holds n mod 2048 seeds", lambda F, n=n: (F.n - 1) // SEG_TILE == (n - 1) // SEG_TILE)
    return c.finish(genomes=True)


TILE_NS = [1, 2, 2047, 2048, 2049, 4095, 4096, 4097, 5 * SEG_TILE - 1, 5 * SEG_TILE + 1, 17 * SEG_TILE - 1,
           17 * SEG_TILE + 1]


def _span_case():
    """one band segment of 300 tiles and 5 seeds between a segment of 10 on the band below and one of 100
    on the band above; 32 seeds an anti-diagonal (dlow 0, 2, .., 62)"""
    c = Case("tiles_span", "tiles")
    k = 300 * SEG_TILE + 5
    c.add(0, 0, 0, MID - 1, dense(10, A0 - 100))
    i = np.arange(k)
    c.add(0, 0, 0, MID, A0 + i // 32, dlow=2 * (i % 32))
    c.add(0, 0, 0, MID + 1, dense(100))
    c.edge("a segment spans more than 300 tiles", lambda F: (np.diff(F.seg.tolist() + [F.n]) >= 300 * SEG_TILE).any())
    c.edge("both triples hold the long segment", lambda F: F.size.tolist()[:2] == [10 + k, k + 100])
    return c.finish(genomes=True)


def _large_case():
    """about 12 M seeds: segments of 1..64 and 65..4000 dense seeds over four contig pairs, bands
    consecutive but for random gaps -- some 6000 tiles in the look-back at once"""
    c = Case("tiles_large", "tiles")
    rng = np.random.default_rng(91)
    n = 0
    for g in range(4):
        band = 300
        while n < (g + 1) * 3_000_000:
            k = int(rng.integers(1, 65)) if rng.random() < 0.6 else int(rng.integers(65, 4001))
            c.add(0, g, 3 - g, band, dense(k))
            n += k
            band += 1 if rng.random() < 0.8 else 2
            assert band < 9000
    c.edge("more than 5000 tiles", lambda F: F.n > 5000 * SEG_TILE)
    c.edge("segment starts at more than 1500 distinct tile offsets",
           lambda F: len(set((F.seg % SEG_TILE).tolist())) > 1500)
    return c.finish()


def _empty_case():
    c = Case("empty", "tiles")
    c.edge("no seed", lambda F: F.n == 0 and len(F.seg) == 0)
    return c.finish(genomes=True)


# ------------------------------------------------------------------------------------------------
#  band adjacency
# ------------------------------------------------------------------------------------------------

def _adjacency_case():
    c = Case("adjacency", "adjacency")
    c.add(0, 0, 0, MID, dense(40))                          # b, b+1: one triple
    c.add(0, 0, 0, MID + 1, dense(40, A0 + 1))
    c.add(0, 0, 0, MID + 10, dense(40))                     # b, b+2: two
    c.add(0, 0, 0, MID + 12, dense(40))
    for q in range(50):                                     # 50 consecutive bands of 20
        c.add(0, 0, 0, MID + 20 + q, dense(20, A0 + 7 * q))
    c.add(0, 0, 0, MID + 100, dense(40))                    # the group's last band, then b+1 of the next pair
    c.add(0, 0, 1, MID + 101, dense(40))
    c.add(0, 3, 3, MID + 200, dense(40))                    # the last strand-N band, then b+1 on strand C
    c.add(1, 3, 3, MID + 201, dense(40))
    c.edge("b, b+1 of one contig pair join", lambda F: F.e[F.at(0, 0, 0, MID)] == F.seg[F.at(0, 0, 0, MID + 1) + 1])
    c.edge("b, b+2 do not", lambda F: F.e[F.at(0, 0, 0, MID + 10)] == F.seg[F.at(0, 0, 0, MID + 12)]
           and F.isnew[F.at(0, 0, 0, MID + 12)])
    c.edge("every inner band of the run is lower and upper half",
           lambda F: all(F.above[F.at(0, 0, 0, MID + 20 + q)] and not F.isnew[F.at(0, 0, 0, MID + 20 + q)]
                         for q in range(1, 49)))
    c.edge("b+1 of the next contig pair does not join",
           lambda F: F.at(0, 0, 1, MID + 101) == F.at(0, 0, 0, MID + 100) + 1 and not F.above[F.at(0, 0, 0, MID + 100)])
    c.edge("b+1 of the other strand does not join",
           lambda F: F.at(1, 3, 3, MID + 201) == F.at(0, 3, 3, MID + 200) + 1 and not F.above[F.at(0, 3, 3, MID + 200)])
    return c.finish(genomes=True)


def _extreme_bands_case():
    top = (1 << LAYOUT[1]) - 1
    c = Case("adjacency_extremes", "adjacency")
    c.add(0, 0, 0, 0, dense(40))
    c.add(0, 0, 0, 1, dense(40))
    c.add(0, 0, 0, top - 1, dense(40))
    c.add(0, 0, 0, top, dense(40))
    c.add(0, 0, 1, 0, dense(40))                            # band 0 of the next pair after the top band
    c.add(0, 0, 1, top, dense(70))
    c.edge("bands 0 and 1 join", lambda F: F.above[F.at(0, 0, 0, 0)])
    c.edge("the top band value is all ones", lambda F: int(F.band.max()) == top)
    c.edge("top-1 and top join", lambda F: F.above[F.at(0, 0, 0, top - 1)])
    c.edge("the top band and band 0 of the next pair do not",
           lambda F: not F.above[F.at(0, 0, 0, top)] and F.isnew[F.at(0, 0, 1, 0)])
    return c.finish()


# ------------------------------------------------------------------------------------------------
#  prefilter bounds
# ------------------------------------------------------------------------------------------------

def _prefilter_case(cm):
    """isolated triples of 63..66 dense seeds, on one band and on two; and triples of the seed bound
    (cm + 79) // 80 and one below it, their seeds 80 anti-diagonals apart: coverage 80 a seed"""
    c = Case("prefilter_cm%d" % cm, "prefilter", chain_min=cm)
    B = (cm + 79) // 80
    band = MID - 100
    for k in (63, 64, 65, 66):
        c.add(0, 0, 0, band, dense(k))
        band += 5
    for lo in (31, 32, 33):
        for up in (32, 33):
            c.add(0, 0, 0, band, dense(lo))
            c.add(0, 0, 0, band + 1, dense(up, A0 + 1))
            band += 5
    spaced = A0 + 80 * np.arange(B)
    c.add(0, 1, 1, MID, spaced)                               # B seeds, one band
    if B >= 2:
        c.add(0, 1, 1, MID + 5, spaced[:B // 2])              # B seeds, two bands
        c.add(0, 1, 1, MID + 6, spaced[B // 2:])
        c.add(0, 1, 1, MID + 10, spaced[:B - 1])              # B - 1
    c.edge("triples of 63, 64, 65 and 66 seeds", lambda F: {63, 64, 65, 66} <= set(F.size[F.scanned].tolist()))
    c.edge("a triple of the seed bound holds a chain and is kept",
           lambda F: F.size[F.at(0, 1, 1, MID)] == B and F.kept[F.at(0, 1, 1, MID)] and F.chain(0, 1, 1, MID) > 0)
    if B >= 2:
        c.edge("a two-band triple of the seed bound holds a chain",
               lambda F: F.size[F.at(0, 1, 1, MID + 5)] == B and F.chain(0, 1, 1, MID + 5) > 0)
        c.edge("one seed below the bound: dropped, and no chain",
               lambda F: F.size[F.at(0, 1, 1, MID + 10)] == B - 1 and not F.kept[F.at(0, 1, 1, MID + 10)]
               and F.chain(0, 1, 1, MID + 10) == 0)
    return c.finish(genomes=True)


PREFILTER_CMS = [1, 80, 81, 170, 2000]


# ------------------------------------------------------------------------------------------------
#  the short-triple scan
# ------------------------------------------------------------------------------------------------

def _short_scan_case():
    """triples of at most 64 seeds, each on its own bands (MID + 10 k), chain_min 170, chain_break 2000"""
    c = Case("short_scan", "short_scan")
    a = A0
    want = []
    K = iter(range(100))

    def put(name, low, up=None, below=None, has=True, mark=0):
        """low / up / below: (anti, plen) of the lower band, the band above and the band below; mark:
        the band (0 lower, -1 below) whose triple must hold a chain or not"""
        b = MID - 300 + 10 * next(K)
        for off, s in ((0, low), (1, up), (-1, below)):
            if s is not None:
                c.add(0, 2, 2, b + off, np.array(s[0]), np.array(s[1]))
        want.append((name, b + mark, has))

    cov170 = ([a, a + 80, a + 160], [40, 40, 5])
    put("coverage exactly chain_min", cov170)
    put("coverage chain_min - 1 (partial branch)", ([a, a + 79, a + 159], [40, 40, 5]), has=False)
    put("overlapping seeds reach chain_min (partial branch)", ([a, a + 50, a + 130], [40, 40, 20]))
    put("a break at exactly ahgh + chain_break", ([a, a + 80, a + 90 + CB], [40, 5, 40]), has=False)
    put("one anti-diagonal before the break", ([a, a + 80, a + 89 + CB], [40, 5, 40]))
    strays = ([a + 5000, a + 5000 + STRAY], [40, 40])
    put("a chain in the lower band only, isnew", cov170, up=strays)
    put("a chain in the lower band only, not isnew", cov170, up=strays, below=strays, has=False)
    put("  ... counted in the triple below, as its upper band", cov170, up=strays, below=strays, mark=-1)
    put("a chain in the upper band only", strays, up=cov170)
    put("a mixed chain", ([a, a + 160], [40, 5]), up=([a + 80], [40]))
    tail = ([a + 5000, a + 5080, a + 5160], [40, 40, 5])
    put("a chain that ends at the triple's last seed, upper band", ([a, a + STRAY], [40, 40]), up=tail)
    put("a chain that ends at the triple's last seed, lower band", tail, up=([a, a + STRAY], [40, 40]))
    put("coverage chain_min - 1 at the triple's last seed", ([a, a + 5000, a + 5079, a + 5159], [40, 40, 40, 5]),
        has=False)
    c.marks = want
    for name, band, has in want:
        c.edge(name, lambda F, band=band, has=has: F.size[F.at(0, 2, 2, band)] <= PREF_LONG
               and F.kept[F.at(0, 2, 2, band)] and (F.chain(0, 2, 2, band) > 0) == has)
    return c.finish(genomes=True)


# ------------------------------------------------------------------------------------------------
#  long-triple order
# ------------------------------------------------------------------------------------------------

def _long_ties_case():
    """40 isolated long triples of three sizes in shuffled order: the launch order falls back to the
    segment index within a size"""
    c = Case("long_ties", "long_order")
    sizes = [70] * 20 + [100] * 10 + [65] * 10
    np.random.default_rng(5).shuffle(sizes)
    for q, k in enumerate(sizes):
        c.add(0, 1, 2, MID - 200 + 5 * q, dense(k))
    c.edge("at least 10 long triples of each of three sizes",
           lambda F: sorted(np.unique(F.size[F.long], return_counts=True)[1].tolist()) == [10, 10, 20])
    return c.finish(genomes=True)


def _long_whole_case(n, bands):
    """one triple that holds every seed, on one band or two: its size n at the top of the sbits field"""
    c = Case("long_whole_%d_%d" % (n, bands), "long_order")
    if bands == 1:
        c.add(0, 0, 0, MID, dense(n))
    else:
        c.add(0, 0, 0, MID, dense(n // 2))
        c.add(0, 0, 0, MID + 1, dense(n - n // 2, A0 + 1))
    c.edge("one long triple holds all %d seeds" % n, lambda F: F.nlong == 1 and F.size[F.lj[0]] == F.n == n)
    c.edge("smax - size = %d" % ((1 << n.bit_length()) - 1 - n),
           lambda F: (1 << F.sbits) - 1 - F.size[F.lj[0]] == (1 << n.bit_length()) - 1 - n)
    return c.finish(genomes=True)


def _densest_case():
    """consecutive bands of 32 and 33 dense seeds in turn on two contig pairs: every segment but each
    pair's last starts a long triple of 65 seeds, within 2 % of the work-list block's bound n / 32 + 2"""
    c = Case("densest", "densest")
    for g in range(2):
        for q in range(1501):
            c.add(0, g, g, MID - 750 + q, dense(32 + q % 2, A0 + 11 * q))
    c.edge("every long triple holds 65 seeds", lambda F: set(F.size[F.long].tolist()) == {65})
    c.edge("long triples reach 98 % of n / 32 + 2", lambda F: F.nlong == 3000 and F.nlong / F.lcap > 0.98)
    return c.finish(genomes=True)


# ------------------------------------------------------------------------------------------------
#  past 2^20 long triples
# ------------------------------------------------------------------------------------------------

BIG_LEN = 4_000_000


def _big_case(nlong):
    """nlong long triples of 65 seeds (bands of 32 and 33 stray seeds in turn) on 16 contig pairs of
    ~4 Mbp a side, none of which holds a chain, and four diverged tubes that align: three on strand N inside
    populated bands, one on strand C on a band of its own (a short work triple)"""
    rng = np.random.default_rng(2020 + nlong)
    A = [rng.integers(0, 4, BIG_LEN + 2 * c, dtype=np.uint8) for c in range(4)]
    B = [rng.integers(0, 4, BIG_LEN + 1 + 2 * c, dtype=np.uint8) for c in range(4)]
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    layout = ol.seed_layout(gA, gB)
    amx, bmx = layout[4], layout[5]
    _, rankA = ol.contig_rank(gA.clen)
    _, rankB = ol.contig_rank(gB.clen)
    c = Case("past_2^20%s" % ("+%d" % (nlong - LONG_SORT_CAP) if nlong > LONG_SORT_CAP else ""), "past_2^20",
             layout=layout)
    mid = bmx >> 6
    per = [nlong // 16 + (1 if g < nlong % 16 else 0) for g in range(16)]
    base = 2_300_000
    for g in range(16):
        nb = per[g] + 1
        bands = mid - nb // 2 + np.arange(nb)
        k = 32 + (np.arange(nb) % 2)
        rep = np.repeat(np.arange(nb), k)
        pos = np.arange(len(rep)) - np.repeat(np.cumsum(k) - k, k)
        c.rows.append(seed_rows(layout, 0, g // 4, g % 4, bands[rep], base + STRAY * pos))
    # the tubes: an exact window of three seeds between 1.5 kbp of 3 % divergence each side
    F, W = 1500, wc.SEED_SPAN + 20
    for q, (comp, i, j, d) in enumerate(((0, 0, 0, 1000), (0, 1, 2, -50_000), (0, 3, 3, 70_000), (1, 1, 1, 0))):
        anti = base + 40 * STRAY + 10_000 * q
        x0 = (anti + d) // 2
        y0 = x0 - d
        Bp = wc.revcomp(B[j]) if comp else B[j]
        left = wc._edit(rng, A[i][x0 - F:x0], 0.025, 0.0025)
        right = wc._edit(rng, A[i][x0 + W:x0 + W + F], 0.025, 0.0025)
        Bp[y0 - len(left):y0] = left
        Bp[y0:y0 + W] = A[i][x0:x0 + W]
        Bp[y0 + W:y0 + W + len(right)] = right
        if comp:
            B[j] = wc.revcomp(Bp)
        rows = [wc.seed_row(comp, rankA[i], rankB[j], x0 + s * wc.SEED_STEP, y0 + s * wc.SEED_STEP, wc.PLEN, len(B[j]))
                for s in range(3)]
        c.rows.append(np.array(rows, dtype=ol.SEED_DT))
    c.edge("%d long triples" % nlong, lambda F: F.nlong == nlong)
    c.edge("the long count is %s 2^20" % ("above" if nlong > LONG_SORT_CAP else "at"),
           lambda F: (F.nlong > LONG_SORT_CAP) == (nlong > LONG_SORT_CAP))
    c.edge("the four tubes are the only chains", lambda F: len(F.oh) == 4)
    c.edge("one short work triple, the strand-C tube", lambda F: len(F.short_work) == 1)
    c.edge("under 36 M seeds", lambda F: F.n < 36_000_000)
    c.edge("a sort key of %d bits" % (int(35_000_000).bit_length() + 21),
           lambda F: F.sbits + F.jbits == int(35_000_000).bit_length() + 21)
    return c.finish(genomes=(A, B))


# ------------------------------------------------------------------------------------------------

BUILDERS = {}
for _n in TILE_NS:
    BUILDERS["tiles_%d_edges" % _n] = (lambda n=_n: _tile_case(n, "edges"))
for _n in (4097, 5 * SEG_TILE + 1, 17 * SEG_TILE - 1):
    BUILDERS["tiles_%d_cross" % _n] = (lambda n=_n: _tile_case(n, "cross"))
BUILDERS["tiles_span"] = _span_case
BUILDERS["empty"] = _empty_case
BUILDERS["adjacency"] = _adjacency_case
BUILDERS["adjacency_extremes"] = _extreme_bands_case
for _cm in PREFILTER_CMS:
    BUILDERS["prefilter_cm%d" % _cm] = (lambda cm=_cm: _prefilter_case(cm))
BUILDERS["short_scan"] = _short_scan_case
BUILDERS["long_ties"] = _long_ties_case
for _n, _b in ((4095, 1), (4096, 1), (4096, 2)):
    BUILDERS["long_whole_%d_%d" % (_n, _b)] = (lambda n=_n, b=_b: _long_whole_case(n, b))
BUILDERS["densest"] = _densest_case
BUILDERS["tiles_large"] = _large_case
BUILDERS["past_2^20"] = lambda: _big_case(LONG_SORT_CAP)
BUILDERS["past_2^20+1"] = lambda: _big_case(LONG_SORT_CAP + 1)

NAMES = list(BUILDERS)
BIG = ("tiles_large", "past_2^20", "past_2^20+1")      # held one at a time

_cases = {}


def case(name):
    if name not in _cases:
        if name in BIG:
            for k in BIG:
                _cases.pop(k, None)
        _cases[name] = BUILDERS[name]()
    return _cases[name]

"""TEST INFRASTRUCTURE (CPU only): crafted table pairs that drive the pair adaptamer merge (merge.cu
adaptamer_merge_kernel) into its corners, a declarative restatement of the merge, and a restatement of the
kernel's per-CTA geometry that says which corner a pair reaches.

A case is a pair of sorted (n, 2) uint64 record tables in the device layout of self_cases.py: T1 holds
both strands (the device compacts it to its forward entries, the oracle's walk runs over all of them), T2
is the table the adaptamers are looked up in.  Every contig of a case has a distinct length above every post
on it, so the same tables can be written as a .gix with a GDB behind it and handed to the reference."""
import os
import re

import numpy as np

import oracle_lib as ol
import self_cases as sc

KMER = 40
TOP = (1 << 24) - 1                       # the last 12-base panel (all T)

# ------------------------------------------------------------------------------------------------
#  the kernel's constants, read from merge.cu so that regimes() follows the kernel
# ------------------------------------------------------------------------------------------------

_MERGE_CU = os.path.join(ol.ROOT, "fastga_b200", "csrc", "merge.cu")


def _kernel_constants():
    src = open(_MERGE_CU).read()
    c = {}
    for name in ("MG_THREADS", "MG_T2CAP", "MG_DCAP", "MG_PCAP"):
        c[name] = int(re.search(r"#define\s+%s\s+(\d+)" % name, src).group(1))
    steps = re.findall(r"if \(ratio <= ([\d.]+)\)\s+rc = merge_launch<(\d+)>", src)
    last = re.search(r"else\s+rc = merge_launch<(\d+)>", src)
    c["tiles"] = [(float(r), int(t)) for r, t in steps] + [(float("inf"), int(last.group(1)))]
    return c


K = _kernel_constants()


# ------------------------------------------------------------------------------------------------
#  cases
# ------------------------------------------------------------------------------------------------

def first_reservation(n1):
    """seeds the merge reserves before its one retry (api.cu seeds_merge_impl), n1 forward T1 entries"""
    return 2 * n1 + n1 // 2 + 1024


class PairCase:
    def __init__(self, name, t1, t2, clen1, clen2, freqs, note):
        self.name, self.freqs, self.note = name, tuple(freqs), note
        self.clen1, self.clen2 = np.asarray(clen1, np.int64), np.asarray(clen2, np.int64)
        self.T1, self.T2 = t1.table(), t2.table()
        for T, clen in ((self.T1, self.clen1), (self.T2, self.clen2)):
            if len(T):
                cont = ((T[:, 0] >> np.uint64(32)) & np.uint64(0x7fff)).astype(np.int64)
                post = (T[:, 0] & np.uint64(0xffffffff)).astype(np.int64)
                assert (post + KMER <= clen[cont]).all(), name
        self.n1 = int((((self.T1[:, 0] >> np.uint64(47)) & np.uint64(1)) == 0).sum()) if len(self.T1) else 0

    def pstart2(self):
        return pstart_of(self.T2)

    @property
    def amx(self):
        return int(self.clen1.max())

    @property
    def bmx(self):
        return int(self.clen2.max())

    def upload_bytes(self, which):
        """(post bytes, contig bytes) of table 1 or 2 as GIXmake chooses them (formats.gix_bytes)"""
        clen = self.clen1 if which == 1 else self.clen2
        pb, cum = 0, 1
        while cum < int(clen.max()):
            cum, pb = cum * 256, pb + 1
        cb, cum = 0, 1
        while cum < 2 * max(len(clen), 8):
            cum, cb = cum * 256, cb + 1
        return pb, cb

    def layout(self):
        """seed record layout of the device (api.cu seed_layout_of) for this pair"""
        anti = int(self.amx + self.bmx).bit_length()
        return (anti, max(anti - 6, 1), int(max(len(self.clen2) - 1, 1)).bit_length(),
                int(max(len(self.clen1) - 1, 1)).bit_length(), self.amx, self.bmx)

    def key_bits(self):
        L = self.layout()
        return 12 + L[0] + L[1] + L[2] + L[3] + 1


def pstart_of(T):
    pre = (T[:, 1] >> np.uint64(40)).astype(np.int64) if len(T) else np.zeros(0, np.int64)
    return np.searchsorted(pre, np.arange((1 << 24) + 1)).astype(np.uint32)


class _Tab:
    """rows of one table: k-mers as 40 bases, strand, contig, post (unique per contig)"""

    def __init__(self, rng, clen):
        self.rng, self.clen = rng, np.asarray(clen, np.int64)
        self.bases, self.signs, self.conts, self.posts = [], [], [], []
        self.used = set()

    def add(self, kmer, sign=0, cont=None, post=None):
        rng = self.rng
        if cont is None:
            cont = int(rng.integers(0, len(self.clen)))
        if post is None:
            while True:
                post = int(rng.integers(0, int(self.clen[cont]) - KMER))
                if (cont, post) not in self.used:
                    break
        self.used.add((cont, post))
        self.bases.append(np.asarray(kmer, np.uint8))
        self.signs.append(sign)
        self.conts.append(cont)
        self.posts.append(post)

    def table(self):
        if not self.bases:
            return np.zeros((0, 2), np.uint64)
        return sc.pack(np.stack(self.bases), np.asarray(self.signs), np.asarray(self.conts), np.asarray(self.posts))


def prefix_bases(p):
    return np.array([(p >> (22 - 2 * k)) & 3 for k in range(12)], np.uint8)


class _Kmers:
    def __init__(self, rng):
        self.rng = rng
        self.taken = set()

    def panel(self, lo=0, hi=TOP + 1):
        """a fresh 12-base panel in [lo, hi) no other part of the case uses"""
        while True:
            p = int(self.rng.integers(lo, hi))
            if p not in self.taken:
                self.taken.add(p)
                return p

    def kmer(self, panel=None):
        k = self.rng.integers(0, 4, KMER).astype(np.uint8)
        k[:12] = prefix_bases(self.panel() if panel is None else panel)
        return k

    def share(self, q, p, base=None):
        """a k-mer sharing exactly p bases with q (q itself at p = 40); base: its base at position p"""
        k = q.copy()
        if p < KMER:
            if base is None:
                base = (int(q[p]) + int(self.rng.integers(1, 4))) % 4
            assert base != q[p]
            k[p] = base
            k[p + 1:] = self.rng.integers(0, 4, KMER - p - 1)
        return k


def _clens(n, top):
    """n distinct decreasing contig lengths, the longest `top`"""
    return np.array([top - 7 * c for c in range(n)], np.int64)


def _setup(seed, n1=8, n2=8, len1=20_000, len2=20_000):
    rng = np.random.default_rng(seed)
    c1, c2 = _clens(n1, len1), _clens(n2, len2)
    return rng, _Kmers(rng), _Tab(rng, c1), _Tab(rng, c2), c1, c2


def freq_edges():
    """T2 blocks of f-1, f and f+1 members for each f: identical 40-mers (the T1 k-mer lands on the block's
    first member), and for the small ones members that share 20 or 35 bases with the T1 k-mer"""
    F = (1, 2, 3, 9, 10, 11, 64, 255)
    rng, km, t1, t2, c1, c2 = _setup(101)
    for f in F:
        for m in (f - 1, f, f + 1):
            if m < 1:
                continue
            for p in ((40, 20, 35) if m <= 3 else (40,)):
                q = km.kmer()
                t1.add(q)
                for _ in range(m):
                    t2.add(km.share(q, p, base=(q[p] + 1) % 4 if p < KMER and m == 1 else None)
                           if p < KMER else q)
    return PairCase("freq_edges", t1, t2, c1, c2, F, "blocks of f-1, f, f+1 members")


def _block_around(km, q, p, left, right):
    """T2 members sharing exactly p bases with q: `left` of them sort before q, `right` after it"""
    assert p < KMER and 0 < q[p] < 3
    out = [km.share(q, p, base=0) for _ in range(left)]
    out += [km.share(q, p, base=3) for _ in range(right)]
    return out


def runs():
    """T2 blocks around the T1 k-mer's insertion point: members on one side only (the insertion point at
    the block's start or end) or on both (the middle), 7, 8, 9, 10, 16 and 17 members a side: the adj-byte
    runs either side of the SIMD compare's eight bytes and of the byte loop"""
    rng, km, t1, t2, c1, c2 = _setup(102)
    for k in (7, 8, 9, 10, 16, 17):
        for left, right in ((0, k), (k, 0), (k, 3), (3, k), (k, k)):
            q = km.kmer()
            q[24] = 1 + (k & 1)
            t1.add(q)
            for x in _block_around(km, q, 24, left, right):
                t2.add(x)
        q = km.kmer()                                   # identical copies: the insertion point at the start
        t1.add(q)
        for _ in range(k):
            t2.add(q)
    return PairCase("runs", t1, t2, c1, c2, (9, 10, 11, 64), "runs of 7..17 members either side")


def plen_sweep():
    """every plen from 12 to 40 with the first difference in the low or the high bit of the base pair, on
    one side or both; and neighbours that share different numbers of bases with the T1 k-mer (the longer
    one decides), either side"""
    rng, km, t1, t2, c1, c2 = _setup(103)
    for p in range(12, KMER + 1):
        for variant in range(4):
            q = km.kmer()
            t1.add(q)
            if p == KMER:
                t2.add(q)
                t2.add(km.share(q, int(rng.integers(12, KMER))))
                continue
            if variant < 2:                              # one member: low / high bit of base p differs
                q[p] = int(rng.integers(0, 4))
                t1.bases[-1] = q
                t2.add(km.share(q, p, base=int(q[p]) ^ (1 + variant)))
            elif variant == 2 and 0 < q[p] < 3:          # a tie: one member either side
                t2.add(km.share(q, p, base=0))
                t2.add(km.share(q, p, base=3))
            else:                                        # p on one side, fewer bases on the other
                lo = int(rng.integers(12, p)) if p > 12 else None
                if q[p] in (0, 3):
                    q[p] = 1
                    t1.bases[-1] = q
                t2.add(km.share(q, p, base=0 if variant & 1 else 3))
                other = 3 if variant & 1 else 0
                if lo is not None and q[lo] != other:
                    t2.add(km.share(q, lo, base=other))
    return PairCase("plen_sweep", t1, t2, c1, c2, (3, 10), "plen 12..40")


def state_machine():
    """dense panels where T1 and T2 k-mers branch off one another at every depth: consecutive T1 entries
    share more, as many and fewer bases than the current match, reverse T1 entries sit between forward
    ones of the same block, and T2 holds duplicates -- the walk of orc_merge takes every branch"""
    rng, km, t1, t2, c1, c2 = _setup(104)

    def tree(root, n, dup):
        out = [root]
        while len(out) < n:
            src = out[int(rng.integers(0, len(out)))]
            if rng.random() < dup:
                out.append(src.copy())
            else:
                out.append(km.share(src, int(rng.integers(12, KMER))))
        return out

    for _ in range(10):
        root = km.kmer()
        a = tree(root, 40, 0.15)
        b = tree(root, 80, 0.25)
        for x in a:
            t1.add(x, int(rng.integers(0, 2)))
            if rng.random() < 0.3:
                t1.add(x, 1 - t1.signs[-1])             # the same k-mer on the other strand
        for x in b:
            t2.add(x, int(rng.integers(0, 2)))
    return PairCase("state_machine", t1, t2, c1, c2, (2, 4, 10, 64), "every branch of orc_merge's walk")


def panels():
    """two TILE-512 tiles: one on panels 0..99 (panel 0 on both sides, T2's first entries), one on the last
    100 panels (T2's last entries, a staged prefix span that ends at 2^24-1 and reads into the index's
    slack); T1 panels empty in T2 next to non-empty ones, and T2 panels with no T1 entry inside a span"""
    rng, km, t1, t2, c1, c2 = _setup(105)
    for base in (0, TOP + 1 - 100):
        ps = list(range(base, base + 100))
        # panels 0 and TOP (the ends) hold several T1 entries and a crowded T2 panel
        for j, p in enumerate(ps):
            kind = 0 if p in (0, TOP) else j % 4         # 0: both, 1: T1 only, 2: T2 only, 3: both, sparse
            nq = 12 if kind == 0 else (3 if kind != 2 else 0)
            qs = []
            for _ in range(nq):
                q = km.kmer(panel=p)
                qs.append(q)
                t1.add(q, int(rng.random() < 0.25))
            if kind in (0, 2, 3):
                for q in (qs or [km.kmer(panel=p)]):
                    for _ in range(int(rng.integers(1, 4))):
                        t2.add(km.share(q, int(rng.integers(12, KMER + 1))))
        while sum(1 for s in t1.signs if s == 0) < (512 if base == 0 else 1024):
            p = int(rng.integers(base + 1, base + 99))
            t1.add(km.kmer(panel=p))
    return PairCase("panels", t1, t2, c1, c2, (2, 10), "panels 0 and 2^24-1, empty panels either side")


def _seeding_entries(km, t1, t2, panels_sorted, seeds_of, rng):
    """one forward T1 entry per panel in panels_sorted; T1 entry i gets a T2 block of seeds_of(i) members
    (0: nothing in its panel)"""
    for i, p in enumerate(panels_sorted):
        q = km.kmer(panel=p)
        t1.add(q)
        m = seeds_of(i)
        if m:
            pl = int(rng.integers(12, KMER + 1))
            x = q if pl == KMER else km.share(q, pl)
            for _ in range(m):
                t2.add(x)


def _filled(km, t2, n2, lo=0, hi=TOP + 1):
    while len(t2.bases) < n2:
        t2.add(km.kmer(panel=km.panel(lo, hi)))


def tile_sizes(n1, n2, seed, round1_only=False, name=None):
    """n1 forward T1 entries on sorted random panels, half of them with a T2 block of 1..3 members in their
    panel, T2 filled to n2 entries in panels of their own.  round1_only: the first tile's entries 0..255
    get no partner, so that its seeds all lie in round 1"""
    rng, km, t1, t2, c1, c2 = _setup(seed)
    ps = sorted(km.panel() for _ in range(n1))

    def seeds_of(i):
        if round1_only and i < 256:
            return 0
        return int(rng.integers(1, 4)) if rng.random() < 0.5 else 0
    _seeding_entries(km, t1, t2, ps, seeds_of, rng)
    _filled(km, t2, n2)
    return PairCase(name or "tiles_%d_%d" % (n1, n2), t1, t2, c1, c2, (2, 3), "n1 %d, n2 %d" % (n1, n2))


#  (n1, n2): the four tiles, exactly at and a hair above each ratio threshold, and last tiles of 1 and
#  TILE-1 entries
TILE_SHAPES = [(1000, 2100), (1000, 2101), (1000, 4200), (1000, 4201), (1000, 8400), (1000, 8401),
               (1025, 1500), (1535, 2000), (513, 2000), (767, 2500), (257, 3000), (383, 3000), (129, 2000),
               (191, 2000)]


def packed_ceiling():
    """-f 255: 512 forward T1 entries of one k-mer against a 254-member T2 block of it: 65024 seeds in each
    round of one TILE-512 CTA, 130048 through the entry-wise write-out (and past the first reservation)"""
    rng, km, t1, t2, c1, c2 = _setup(106, len1=200_000)
    q = km.kmer()
    for _ in range(512):
        t1.add(q)
    for _ in range(254):
        t2.add(q)
    return PairCase("packed_ceiling", t1, t2, c1, c2, (255,), "65024 seeds a round")


def staging():
    """TILE-64 tiles (T2 is filled to more than 8.4 times T1 in panels outside every tile) whose T2 slice
    holds exactly 0, 1, 1152 and 1153 entries, whose prefix span is 512 and 513 index words (the first
    panel a multiple of 4), whose span ends at panel 2^24-1, and whose seed totals are exactly 1536 and 1537
    (at -f 64 and 255)"""
    rng, km, t1, t2, c1, c2 = _setup(107)
    F = (3, 10, 64, 255)
    band = (1 << 24) // 16                            # tile i lives in panels [i*band, (i+1)*band)
    bands = []

    def tile_panels(i, n, span=None):
        lo = i * band
        if span is None:
            return sorted(km.panel(lo, lo + 4000) for _ in range(n))
        first = lo - lo % 4
        mid = sorted(km.panel(first + 1, first + span) for _ in range(n - 2))
        km.taken.update((first, first + span))
        return [first] + mid + [first + span]

    def block_sizes():                                # blocks around every f (T2 members per T1 entry)
        return [m for f in F[:3] for m in (f - 1, f, f + 1)]

    # tile 0: no T2 entry in its span
    for p in tile_panels(0, 64):
        t1.add(km.kmer(panel=p))
    # tile 1: one T2 entry in its span
    ps = tile_panels(1, 64)
    for j, p in enumerate(ps):
        q = km.kmer(panel=p)
        t1.add(q)
        if j == 30:
            t2.add(km.share(q, 30))
    # tiles 2 and 3: slices of 1152 and 1153 entries -- blocks around every f, the rest in panels of the span
    #                that no T1 entry uses
    for i, nsl in ((2, 1152), (3, 1153)):
        ps = tile_panels(i, 64)
        sizes = block_sizes()
        start = len(t2.bases)
        for j, p in enumerate(ps):
            q = km.kmer(panel=p)
            t1.add(q)
            if j < len(sizes):
                for _ in range(sizes[j]):
                    t2.add(q)
            elif j % 3 == 0:
                t2.add(km.share(q, int(rng.integers(12, 40))))
        while len(t2.bases) - start < nsl:
            t2.add(km.kmer(panel=km.panel(ps[0] + 1, ps[-1])))
    # tiles 4 and 5: prefix spans of 512 and 513 index words (pB - pA = 510, 511)
    for i, span in ((4, 510), (5, 511)):
        for j, p in enumerate(tile_panels(i, 64, span)):
            q = km.kmer(panel=p)
            t1.add(q)
            if j % 2 == 0:
                t2.add(km.share(q, int(rng.integers(12, 41))))
    # tiles 6 and 7: CTA totals of 1536 = 64 x 24 and 1537 = 63 x 24 + 25
    for i, extra in ((6, 0), (7, 1)):
        p0, p1 = km.panel(i * band, i * band + 1000), km.panel(i * band + 1000, i * band + 2000)
        q, r = km.kmer(panel=p0), km.kmer(panel=p1)
        for _ in range(64 - extra):
            t1.add(q)
        for _ in range(24):
            t2.add(q)
        if extra:
            t1.add(r)
            for _ in range(25):
                t2.add(r)
    # tile 8 (the last, 40 entries): a staged span that ends at panel 2^24-1
    for j, p in enumerate([TOP - 200 + 5 * k for k in range(39)] + [TOP]):
        km.taken.add(p)
        q = km.kmer(panel=p)
        t1.add(q)
        t2.add(km.share(q, 12 + j % 29))
    assert len(t1.bases) == 8 * 64 + 40
    _filled(km, t2, 9 * len(t1.bases), 9 * band, 15 * band)
    return PairCase("staging", t1, t2, c1, c2, F, "slices of 0/1/1152/1153, spans of 512/513 words, totals 1536/1537")


def strands():
    """T2 blocks on mixed strands, a palindromic 40-mer (one post on both strands, with further copies), and
    reverse T1 entries of the same k-mers as forward ones"""
    rng, km, t1, t2, c1, c2 = _setup(108)
    for m in (2, 3, 5, 9):
        for signs in ([0, 1] * m, [1] * m, [0] * (m - 1) + [1]):
            q = km.kmer()
            t1.add(q, 0)
            t1.add(q, 1)
            for s in signs[:m]:
                t2.add(q, s)
    for m in (2, 3, 6):                               # palindromes: post x on both strands
        q = km.kmer()
        t1.add(q, 0)
        t2.add(q, 0, cont=0, post=1000 + m)
        t2.add(q, 1, cont=0, post=1000 + m)
        for _ in range(m - 2):
            t2.add(q, int(rng.integers(0, 2)))
    return PairCase("strands", t1, t2, c1, c2, (3, 4, 10), "mixed strands, palindromes")


def no_forward():
    """a T1 with reverse entries only: nothing left after the compaction (n1 = 0)"""
    rng, km, t1, t2, c1, c2 = _setup(109)
    for _ in range(50):
        q = km.kmer()
        t1.add(q, 1)
        t2.add(q)
    return PairCase("no_forward", t1, t2, c1, c2, (10,), "n1 = 0")


def forward_only():
    """a T1 that is forward-only already"""
    rng, km, t1, t2, c1, c2 = _setup(110)
    for _ in range(300):
        q = km.kmer()
        t1.add(q, 0)
        for _ in range(int(rng.integers(0, 4))):
            t2.add(km.share(q, int(rng.integers(12, 41))), int(rng.integers(0, 2)))
    return PairCase("forward_only", t1, t2, c1, c2, (3, 10), "T1 forward-only")


def widths():
    """300 contigs a side (2-byte contig fields), the longest contig past 2^24 with posts above 2^24 on it
    (4-byte posts), and so a seed key of 77 bits"""
    rng = np.random.default_rng(111)
    km = _Kmers(rng)
    c1 = np.concatenate([[(1 << 24) + 9000], 2000 - 3 * np.arange(299)]).astype(np.int64)
    c2 = np.concatenate([[(1 << 24) + 7000], 2100 - 3 * np.arange(299)]).astype(np.int64)
    t1, t2 = _Tab(rng, c1), _Tab(rng, c2)
    for i in range(600):
        q = km.kmer()
        big = i % 3 == 0
        t1.add(q, 0, cont=0 if big else int(rng.integers(1, 300)),
               post=int(rng.integers(1 << 24, (1 << 24) + 8000)) if big else None)
        for j in range(int(rng.integers(1, 4))):
            big2 = (i + j) % 2 == 0
            t2.add(km.share(q, int(rng.integers(12, 41))) if j else q, int(rng.integers(0, 2)),
                   cont=0 if big2 else int(rng.integers(1, 300)),
                   post=int(rng.integers(1 << 24, (1 << 24) + 6000)) if big2 else None)
    return PairCase("widths", t1, t2, c1, c2, (3, 10), "2-byte contigs, 4-byte posts, 77-bit seed key")


def overflow():
    """blocks of 9 identical T2 entries under every T1 entry at -f 10: 9 seeds per entry, more than the
    2 n1 + n1/2 + 1024 the merge first reserves"""
    rng, km, t1, t2, c1, c2 = _setup(112)
    for _ in range(400):
        q = km.kmer()
        t1.add(q)
        for _ in range(9):
            t2.add(q)
    return PairCase("overflow", t1, t2, c1, c2, (10,), "seeds > 2 n1 + n1/2 + 1024")


CASES = {"freq_edges": freq_edges, "runs": runs, "plen_sweep": plen_sweep, "state_machine": state_machine,
         "panels": panels, "packed_ceiling": packed_ceiling, "staging": staging, "strands": strands,
         "no_forward": no_forward, "forward_only": forward_only, "widths": widths, "overflow": overflow}
for _k, (_n1, _n2) in enumerate(TILE_SHAPES):
    CASES["tiles_%d_%d" % (_n1, _n2)] = (lambda a, b, s: lambda: tile_sizes(a, b, s))(_n1, _n2, 200 + _k)
CASES["tiles_round1"] = lambda: tile_sizes(1000, 1500, 199, round1_only=True, name="tiles_round1")

_cache = {}


def case(name):
    if name not in _cache:
        _cache[name] = CASES[name]()
    return _cache[name]


# ------------------------------------------------------------------------------------------------
#  the declarative merge (SURVEY A.3), by brute force inside each panel
# ------------------------------------------------------------------------------------------------

def bases_of(T):
    """(n, 40) bases of the k-mers of device-layout records"""
    out = np.zeros((len(T), KMER), np.uint8)
    hi, lo = T[:, 1], T[:, 0]
    for k in range(32):
        out[:, k] = (hi >> np.uint64(62 - 2 * k)) & np.uint64(3)
    for k in range(8):
        out[:, 32 + k] = (lo >> np.uint64(62 - 2 * k)) & np.uint64(3)
    return out


def lcp_matrix(A, B):
    """shared leading bases of every k-mer of A (k, 40) with every one of B (m, 40)"""
    return np.cumprod(A[:, None, :] == B[None, :, :], axis=2).sum(axis=2)


def declarative_merge(T1, T2, pstart2, freq):
    """for every forward T1 entry whose panel is non-empty in T2: plen = the most bases it shares with a T2
    entry of the panel, R = the T2 entries sharing plen bases; |R| < freq seeds (plen, e1, e2) for all e2 in R,
    strand C iff e2 is a reverse entry.  Returns (seeds as ol.SEED_DT, sum of plen)"""
    if len(T1) == 0 or len(T2) == 0:
        return np.zeros(0, ol.SEED_DT), 0
    fwd = np.flatnonzero(((T1[:, 0] >> np.uint64(47)) & np.uint64(1)) == 0)
    pre = (T1[fwd, 1] >> np.uint64(40)).astype(np.int64)
    B1, B2 = bases_of(T1), bases_of(T2)
    rows = []
    for p in np.unique(pre):
        lo, hi = int(pstart2[p]), int(pstart2[p + 1])
        if lo == hi:
            continue
        mine = fwd[pre == p]
        L = lcp_matrix(B1[mine], B2[lo:hi])
        plen = L.max(axis=1)
        for r, i in enumerate(mine):
            R = np.flatnonzero(L[r] == plen[r]) + lo
            if len(R) >= freq:
                continue
            for j in R:
                rows.append((plen[r], (int(T2[j, 0]) >> 47) & 1, (int(T1[i, 0]) >> 32) & 0x7fff,
                             (int(T2[j, 0]) >> 32) & 0x7fff, int(T1[i, 0]) & 0xffffffff,
                             int(T2[j, 0]) & 0xffffffff))
    out = np.array(rows, dtype=ol.SEED_DT) if rows else np.zeros(0, ol.SEED_DT)
    return out, int(out["plen"].astype(np.int64).sum())


# ------------------------------------------------------------------------------------------------
#  the kernel's geometry
# ------------------------------------------------------------------------------------------------

ROWS = ("tile512", "tile256", "tile128", "tile64",
        "two_rounds", "round1_only", "packed_ceiling",
        "staged", "direct",
        "sp_staged", "sp_l1", "sp_top_panel",
        "desc_out", "entry_out", "total_1536", "total_1537",
        "slice_0", "slice_1", "slice_1152", "slice_1153", "words_512", "words_513",
        "run7", "run8", "run9", "run16", "run17", "byte_loop_f10", "byte_loop_f11", "no_loop_f9",
        "ins_start", "ins_middle", "ins_end", "nbr_other_panel", "slice_start", "slice_end",
        "table_start", "table_end", "prefix0", "prefix_top",
        "plen_hi", "plen_lo", "plen_base39", "plen40", "plen_tie",
        "overflow")


def regimes(T1, T2, pstart2, freq):
    """The geometry the kernel gives a pair at freq: the tile from the forward count, and per CTA
    merge_ranges_kernel's (pA, pB, lo2, nsl), the staged / sp decisions, the seed totals of the CTA and of
    its two rounds and the write-out; per forward T1 entry (in CTA order) its insertion point, the LCPs of
    its neighbours, plen, the block members left and right of the insertion point and whether the byte loop
    runs.  Returns (ctas, entries, reached) -- reached: the ROWS this pair reaches at freq."""
    fwd = T1[((T1[:, 0] >> np.uint64(47)) & np.uint64(1)) == 0] if len(T1) else T1
    n1, n2 = len(fwd), len(T2)
    reached = set()
    if n1 == 0:
        return [], [], reached
    ratio = float(n2 if n2 > 0 else 1) / float(n1)
    tile = next(t for r, t in K["tiles"] if ratio <= r)
    reached.add("tile%d" % tile)
    B1, B2 = bases_of(fwd), bases_of(T2)
    adj = np.zeros(n2 + 1, np.int64)                   # adj[i]: LCP of T2 entries i-1 and i, 0 at both ends
    if n2 > 1:
        adj[1:n2] = np.cumprod(B2[1:] == B2[:-1], axis=1).sum(axis=1)
    pre1 = (fwd[:, 1] >> np.uint64(40)).astype(np.int64)
    pre2 = (T2[:, 1] >> np.uint64(40)).astype(np.int64) if n2 else np.zeros(0, np.int64)
    key2 = [bytes(b) for b in B2]
    ctas, entries = [], []
    T = K["MG_THREADS"]
    total_all = 0
    for b0 in range(0, n1, tile):
        b1 = min(b0 + tile, n1) - 1
        pA, pB = int(pre1[b0]), int(pre1[b1])
        lo2, nsl = int(pstart2[pA]), int(pstart2[pB + 1]) - int(pstart2[pA])
        staged = nsl <= K["MG_T2CAP"]
        words = (pA & 3) + (pB - pA) + 2
        sp = staged and nsl > 0 and ((words + 3) & ~3) <= K["MG_PCAP"]
        rounds = [0, 0]
        for j in range(b0, b1 + 1):
            p = pre1[j]
            lo, hi = int(pstart2[p]), int(pstart2[p + 1])
            k1 = bytes(B1[j])
            a = lo + int(np.searchsorted(key2[lo:hi], k1)) if hi > lo else lo
            e = dict(j=j, cta=len(ctas), a=a, lo=lo, hi=hi, ll=0, lr=0, m=0, cnt=0, runL=0, runR=0,
                     loopL=False, loopR=False)
            if hi > lo:
                ll = int(np.cumprod(B1[j] == B2[a - 1]).sum()) if a > lo else 0
                lr = int(np.cumprod(B1[j] == B2[a]).sum()) if a < hi else 0
                m = max(ll, lr)
                runL = runR = 0
                if ll == m:
                    x = a - 1
                    runL = 1
                    while x > lo and adj[x] >= m:
                        x, runL = x - 1, runL + 1
                if lr == m:
                    x = a
                    runR = 1
                    while x + 1 < hi and adj[x + 1] >= m:
                        x, runR = x + 1, runR + 1
                size = runL + runR
                e.update(ll=ll, lr=lr, m=m, runL=runL, runR=runR, size=size, cnt=size if size < freq else 0,
                         loopL=staged and runL - 1 >= 8 and freq > 9, loopR=staged and runR - 1 >= 8 and freq > 9)
                e["tie"] = ll == lr
            rounds[(j - b0) // T if tile >= T else 0] += e["cnt"]
            entries.append(e)
        total = rounds[0] + rounds[1]
        total_all += total
        fast = staged and total <= K["MG_DCAP"]
        ctas.append(dict(pA=pA, pB=pB, lo2=lo2, nsl=nsl, staged=staged, words=words, sp=sp, rounds=rounds,
                         total=total, fast=fast, nt1=b1 - b0 + 1))
    for c in ctas:
        reached.add("staged" if c["staged"] else ("direct" if c["total"] else "direct_noseed"))
        if c["staged"] and c["nsl"] > 0:
            reached.add("sp_staged" if c["sp"] else "sp_l1")
            if c["sp"] and c["pB"] == TOP:
                reached.add("sp_top_panel")
        if c["staged"] and c["total"]:
            reached.add("desc_out" if c["fast"] else "entry_out")
        if c["total"] in (1536, 1537) and c["staged"]:
            reached.add("total_%d" % c["total"])
        if c["nsl"] in (0, 1, 1152, 1153):
            reached.add("slice_%d" % c["nsl"])
        if c["words"] in (512, 513) and c["staged"] and c["nsl"] > 0:
            reached.add("words_%d" % c["words"])
        if tile >= 2 * T:
            if c["rounds"][0] and c["rounds"][1]:
                reached.add("two_rounds")
            if c["rounds"][1] and not c["rounds"][0]:
                reached.add("round1_only")
            if max(c["rounds"]) == 254 * 256:
                reached.add("packed_ceiling")
    for e in entries:
        if e["m"] < 12:
            continue
        c = ctas[e["cta"]]
        for side in ("runL", "runR"):
            if e[side] in (7, 8, 9, 16, 17) and c["staged"]:
                reached.add("run%d" % e[side])
        if e["loopL"] or e["loopR"]:
            reached.add("byte_loop_f%d" % freq)
        if freq == 9 and c["staged"] and max(e["runL"], e["runR"]) >= 9:
            reached.add("no_loop_f9")
        if e["cnt"] == 0:
            continue
        reached.add("ins_middle" if e["runL"] and e["runR"] else ("ins_start" if e["runR"] else "ins_end"))
        a, lo, hi = e["a"], e["lo"], e["hi"]
        if (a == lo and a > c["lo2"]) or (a == hi and a < c["lo2"] + c["nsl"]):
            reached.add("nbr_other_panel")
        if a == c["lo2"] and e["runR"]:
            reached.add("slice_start")
        if a == c["lo2"] + c["nsl"] and e["runL"]:
            reached.add("slice_end")
        if a == 0:
            reached.add("table_start")
        if a == n2:
            reached.add("table_end")
        p = int(pre1[e["j"]])
        if p == 0:
            reached.add("prefix0")
        if p == TOP:
            reached.add("prefix_top")
        m = e["m"]
        reached.add("plen_hi" if m < 32 else ("plen_lo" if m < 40 else "plen40"))
        if m == 39:
            reached.add("plen_base39")
        if e["tie"] and e["runL"] and e["runR"] and m < 40:
            reached.add("plen_tie")
    if total_all > first_reservation(n1):
        reached.add("overflow")
    return ctas, entries, reached


def regimes_of(c, freq):
    return regimes(c.T1, c.T2, c.pstart2(), freq)


# ------------------------------------------------------------------------------------------------
#  the reference's run on a case
# ------------------------------------------------------------------------------------------------

def _write_side(wd, root, T, clen, rng):
    """<root>.gix with one .ktab part, and <root>.1gdb (FAtoGDB) of random contigs of lengths clen"""
    from fastga_b200 import formats
    pb = 0
    cum = 1
    while cum < int(clen.max()):
        cum, pb = cum * 256, pb + 1
    cb, cum = 0, 1
    while cum < 2 * max(len(clen), 8):
        cum, cb = cum * 256, cb + 1
    pstart = pstart_of(T)
    ent = formats.ktab_entries_from_table(T, pb, cb, [0])
    maxpre = int(np.diff(pstart.astype(np.int64)).max()) if len(T) else 0
    formats.write_gix(os.path.join(wd, root + ".gix"), KMER, pstart[1:].astype(np.int64), pb, cb, maxpre,
                      np.arange(len(clen), dtype=np.int32), ent, [len(T)])
    scaf = [("%s_%d" % (root, c), rng.integers(0, 4, int(n)).astype(np.uint8)) for c, n in enumerate(clen)]
    formats.write_fasta(os.path.join(wd, root + ".fasta"), scaf)
    ol.run_ref(["FAtoGDB", root + ".fasta"], cwd=wd)


def ref_merge(c, freqs):
    """`FastGA -v -f<f>` on the case's two tables written as .gix (with a GDB of random contigs of the
    case's lengths behind each): {f: {"seeds": N, "avelen": X}}"""
    import tempfile
    out = {}
    with tempfile.TemporaryDirectory() as wd:
        rng = np.random.default_rng(7)
        _write_side(wd, "A", c.T1, c.clen1, rng)
        _write_side(wd, "B", c.T2, c.clen2, rng)
        for f in freqs:
            log = ol.run_ref(["FastGA", "-v", "-T4", "-P" + wd, "-1:ref", "-f%d" % f, "A", "B"], cwd=wd)
            # no seeds: the reference prints "ave. len = -nan"
            m = re.search(r"Total seeds = ([\d,]+), ave\. len = (\S+),", log)
            n = int(m.group(1).replace(",", ""))
            out[str(f)] = {"seeds": n, "avelen": float(m.group(2)) if n else None}
    return out


def reference_merge(c):
    """the reference's seed count and average length of case c at each of its f (stored golden)"""
    return ol.reference("pair_merge/" + c.name, ol.digest(c.T1, c.T2, c.clen1, c.clen2, list(c.freqs)),
                        lambda: ref_merge(c, c.freqs))

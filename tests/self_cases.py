"""TEST INFRASTRUCTURE (CPU only): inputs that drive SELF mode (`FastGA A`) into its corners.

Crafted self TABLES -- sorted (n, 2) uint64 k-mer records as the device holds them (hi = bases 0..31, base 0
on top; lo = bases 32..39 in bits 63..48, the strand in bit 47, the contig in bits 46..32, the post in bits
31..0), for lib.DeviceGix.upload, which builds the prefix index on the device.  Each table is built from
BLOCKS: runs of entries that share exactly `plen` bases with each other and fewer with anything else, so the
self merge makes a block of m members into m (m - 1) seeds when m < freq and none otherwise.

Self GENOMES -- the straddle genome reaches the branch of align_contigs that makes no call for a chain across
the main diagonal (FastGA.c:3262); the divergence genome reaches it right after a call that ended far into
another contig, so the reference's tube advance (the stale bepos of that call) and the CUDA path's (0) keep
different records."""
import numpy as np

import oracle_lib as ol
from fastga_b200 import formats, synth

KMER = 40
FREQS = (1, 2, 3, 10, 64, 255)
AMX = 4_000_000                      # contig length the tables claim: posts lie below it


class Block:
    """m entries sharing exactly plen bases (m <= 4 when plen < 40: they differ at base plen)"""

    def __init__(self, bases, signs, conts, posts, plen):
        self.bases, self.signs, self.conts, self.posts, self.plen = bases, signs, conts, posts, plen

    @property
    def m(self):
        return len(self.posts)


class TableCase:
    def __init__(self, name, blocks, singles, ncontig, note):
        self.name, self.blocks, self.ncontig, self.note = name, blocks, ncontig, note
        bases = [b.bases for b in blocks] + [singles[0]]
        signs = [b.signs for b in blocks] + [singles[1]]
        conts = [b.conts for b in blocks] + [singles[2]]
        posts = [b.posts for b in blocks] + [singles[3]]
        self.tab = pack(np.concatenate(bases), np.concatenate(signs), np.concatenate(conts),
                        np.concatenate(posts))
        self.n = len(self.tab)

    def pstart(self):
        """lower bound of every 12-base panel (the index the device builds)"""
        pre = (self.tab[:, 1] >> np.uint64(40)).astype(np.int64)
        return np.searchsorted(pre, np.arange((1 << 24) + 1)).astype(np.uint32)

    def seeding_posts(self, freq):
        """posts of the blocks that seed at freq, and of those that do not"""
        yes = [b.posts for b in self.blocks if 2 <= b.m < freq]
        no = [b.posts for b in self.blocks if b.m >= freq]
        cat = lambda x: np.concatenate(x) if x else np.zeros(0, np.int64)
        return cat(yes), cat(no)


def pack(bases, signs, conts, posts):
    """(n, 40) bases, strands, contigs, posts -> sorted (n, 2) uint64 records [lo, hi]"""
    b = bases.astype(np.uint64)
    hi = np.zeros(len(b), np.uint64)
    for k in range(32):
        hi |= b[:, k] << np.uint64(62 - 2 * k)
    lo = np.zeros(len(b), np.uint64)
    for k in range(8):
        lo |= b[:, 32 + k] << np.uint64(62 - 2 * k)
    lo |= (signs.astype(np.uint64) << np.uint64(47)) | (conts.astype(np.uint64) << np.uint64(32)) | \
        posts.astype(np.uint64)
    tab = np.stack([lo, hi], axis=1)
    order = np.lexsort((lo, hi))
    tab = np.ascontiguousarray(tab[order])
    assert not (tab[1:] == tab[:-1]).all(axis=1).any()
    return tab


class _Maker:
    """draws blocks with fresh random prefixes and globally unique posts"""

    def __init__(self, seed, ncontig=4):
        self.rng = np.random.default_rng(seed)
        self.ncontig = ncontig
        self.next_post = 0
        self.posts = self.rng.permutation(AMX - KMER)

    def _posts(self, m):
        p = self.posts[self.next_post:self.next_post + m]
        self.next_post += m
        return p.astype(np.int64)

    def block(self, m, plen, prefix=None, signs=None, conts=None):
        rng = self.rng
        base = rng.integers(0, 4, KMER, dtype=np.uint8)
        if prefix is not None:
            base[:len(prefix)] = prefix
        bases = np.tile(base, (m, 1))
        if plen < KMER:
            assert m <= 4
            bases[:, plen] = rng.permutation(4)[:m]
            bases[:, plen + 1:] = rng.integers(0, 4, (m, KMER - plen - 1))
        if signs is None:
            signs = rng.integers(0, 2, m)
        if conts is None:
            conts = rng.integers(0, self.ncontig, m)
        return Block(bases, np.asarray(signs), np.asarray(conts), self._posts(m), plen)

    def singles(self, n, prefix=None):
        bases = self.rng.integers(0, 4, (n, KMER), dtype=np.uint8)
        if prefix is not None:
            bases[:, :len(prefix)] = prefix
        return (bases, self.rng.integers(0, 2, n), self.rng.integers(0, self.ncontig, n), self._posts(n))


def _no_singles():
    return (np.zeros((0, KMER), np.uint8), np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64))


def freq_blocks():
    """blocks of freq-1, freq and freq+1 members at freq 1, 2, 3, 10, 64, 255: identical 40-mers, and at
    12, 20, 31, 32, 33 and 39 shared bases where the block is small enough; plus, per freq, a block three
    times longer than freq, so that an entry deep inside it meets the bounded walk"""
    M = _Maker(1)
    blocks = []
    for f in FREQS:
        for m in (f - 1, f, f + 1, 3 * f + 5):
            if m < 2:
                continue
            blocks.append(M.block(m, KMER))
            if m <= 4:
                for p in (12, 20, 31, 32, 33, 39):
                    blocks.append(M.block(m, p))
    return TableCase("freq_blocks", blocks, M.singles(300), M.ncontig, "blocks around every freq")


def plen_sweep():
    """every plen from 12 to 40, blocks of 2, 3 and 4: the first difference in the hi word (plen < 32), in
    the lo word (32..39), and none (40-base ties)"""
    M = _Maker(2)
    blocks = [M.block(m, p) for p in range(12, KMER + 1) for m in (2, 3, 4)]
    return TableCase("plen_sweep", blocks, M.singles(200), M.ncontig, "plen 12..40")


def panels():
    """panel 0 (all A) and panel 2^24-1 (all T), each holding several blocks, so that blocks sit first and
    last in their panel and next to blocks that share 12 to 20 bases with them; singleton panels"""
    M = _Maker(3)
    blocks = []
    for fill in (0, 3):
        pre = np.full(12, fill, np.uint8)
        for share in (12, 13, 16, 20):
            sub = np.concatenate([pre, M.rng.integers(0, 4, share - 12, dtype=np.uint8)])
            for m, p in ((2, 40), (3, 25), (4, 36), (9, 40)):
                if p > share:
                    blocks.append(M.block(m, p, prefix=sub))
    singles = M.singles(400)
    return TableCase("panels", blocks, singles, M.ncontig, "panels 0 and 2^24-1, crowded and singleton panels")


def strands():
    """blocks whose members lie on both strands, including a palindromic 40-mer: one post on both strands
    (the same k-mer read either way), with further copies on either strand"""
    M = _Maker(4)
    blocks = []
    for m in (2, 3, 5, 9, 30):
        for signs in ([0, 1] * m, [1] * m, [0] * (m - 1) + [1]):
            blocks.append(M.block(m, KMER, signs=signs[:m]))
    for p in (14, 33):
        blocks.append(M.block(4, p, signs=[0, 1, 0, 1]))
    # palindromes: posts x, x (both strands) and further copies
    for m in (2, 3, 6):
        b = M.block(m, KMER)
        b.posts[1] = b.posts[0]
        b.conts[1] = b.conts[0]
        b.signs[0], b.signs[1] = 0, 1
        blocks.append(b)
    return TableCase("strands", blocks, M.singles(100), M.ncontig, "mixed strands, palindromes")


def sized(n):
    """exactly n entries: blocks of 2..9 members, then singletons up to n"""
    M = _Maker(10 + n)
    blocks, k = [], 0
    while True:
        m = int(M.rng.integers(2, 10))
        if k + m > n - 20:
            break
        blocks.append(M.block(m, KMER if m > 4 else int(M.rng.integers(12, KMER + 1))))
        k += m
    return TableCase("n%d" % n, blocks, M.singles(n - k), M.ncontig, "n = %d" % n)


def large():
    """over a million entries: singletons and 20000 blocks of 2..12 (sharing 20 bases or more: a random
    single sharing as many with a block is unlikely)"""
    M = _Maker(5)
    blocks = [M.block(m, KMER if m > 4 else int(M.rng.integers(20, KMER + 1)))
              for m in M.rng.integers(2, 13, 20_000).tolist()]
    return TableCase("large", blocks, M.singles(1_050_000), M.ncontig, "n > 1 M")


def overflow():
    """blocks of 9 at freq 10: 8 seeds per entry, more than the 2n + 1024 the merge first reserves"""
    M = _Maker(6)
    blocks = [M.block(9, KMER) for _ in range(400)]
    return TableCase("overflow", blocks, _no_singles(), M.ncontig, "seeds > 2n + 1024")


def contigs2b():
    """contig numbers up to 4999: 2-byte contig fields, and a seed key wider than 64 bits"""
    M = _Maker(7, ncontig=5000)
    blocks = [M.block(int(m), KMER if m > 4 else 24) for m in M.rng.integers(2, 12, 800).tolist()]
    return TableCase("contigs2b", blocks, M.singles(2000), M.ncontig, "2-byte contig fields")


TABLES = {"freq_blocks": freq_blocks, "plen_sweep": plen_sweep, "panels": panels, "strands": strands,
          "n255": lambda: sized(255), "n256": lambda: sized(256), "n257": lambda: sized(257), "large": large,
          "overflow": overflow, "contigs2b": contigs2b}


def table(name):
    return TABLES[name]()


# ------------------------------------------------------------------------------------------------
#  self genomes
# ------------------------------------------------------------------------------------------------

def _tandem(rng, unit_len, total, div):
    unit = rng.integers(0, 4, unit_len, dtype=np.uint8)
    parts, n = [], 0
    while n < total:
        parts.append(synth._small_mutations(rng, unit, div))
        n += len(parts[-1])
    return np.concatenate(parts)


def straddle_genome():
    """a 60 kbp flank, 6 kbp of a 12..45-base unit copied with 8..15 % small mutations, a 40 kbp flank; and
    a second random contig.  The array's chains on both sides of the main diagonal come out as one chain
    across it whenever its two bands straddle the diagonal, and as calls with lbord or hbord elsewhere."""
    rng = np.random.default_rng(1)
    c0 = np.concatenate([rng.integers(0, 4, 60_000, dtype=np.uint8),
                         _tandem(rng, int(rng.integers(12, 46)), 6000, float(rng.uniform(0.08, 0.15))),
                         rng.integers(0, 4, 40_000, dtype=np.uint8)])
    return [c0, rng.integers(0, 4, 30_001, dtype=np.uint8)]


def divergence_genome():
    """Contig Y: 300 bases, nine exact copies of a 13-base unit, 20 kbp, a 100-base unit twice (2 %
    diverged), 20 kbp.  Contig X, the longest (so Y's chains against X come first in scan order): 150 kbp,
    then a copy of Y[5000:8000], filled to a length of 50 mod 64 -- which puts Y's main diagonal 50
    diagonals into its band.  In scan order, Y against itself starts with the band pair below the main
    diagonal's band; it holds the 13-periodic chain (on both sides of the diagonal: no call) and, 20 kbp
    later, the 100-base repeat's chain below the diagonal.  The last call before the straddle is Y against
    X, ending 153 kbp into X: the reference advances the straddle's tube to that bepos, past the repeat's
    chain, which it then skips; advancing with 0 aligns it."""
    rng = np.random.default_rng(2)
    R = lambda n: rng.integers(0, 4, n, dtype=np.uint8)
    u1, u2 = R(13), R(100)
    Y = np.concatenate([R(300), np.tile(u1, 9), R(20_000), u2, synth._small_mutations(rng, u2, 0.02), R(20_000)])
    xl = 200_000 - (200_000 % 64) + 50
    X = np.concatenate([R(150_000), synth._small_mutations(rng, Y[5000:8000], 0.03)])
    return [np.concatenate([X, R(xl - len(X))]), Y]


GENOMES = {"straddle": straddle_genome, "divergence": divergence_genome}
DIVERGENT_RECORDS = 1          # records the zero advance keeps on the divergence genome that the reference does not


class SelfRun:
    """the oracle's SELF-mode search of a genome from given seed records (by default its own merge), with
    every Local_Alignment call logged and the straddle advanced as straddle_zero says"""

    def __init__(self, G, recs=None, layout=None, perm=None, straddle_zero=True):
        self.G = G
        self.g = formats.genome_from_arrays(G)
        g = self.g
        if recs is None:
            perm, rank = ol.contig_rank(g.clen)
            t, s = ol.gix_build(g, rank)
            layout = ol.seed_layout(g, g)
            recs = ol.seed_records(ol.self_merge(t, s)[0], layout)
        self.recs, self.layout, self.perm = recs, layout, np.asarray(perm, np.int32)
        with ol.self_search(straddle_zero):
            self.ov, self.tp, self.nhit, self.calls, self.passes = ol.search_calls(recs, layout, g, g, self.perm,
                                                                                    self.perm, g.freq)
            self.counters = ol.self_counters()

    def call_args(self):
        """the calls as ol.ref_local_alignments takes them: (framed a, framed b, comp, low, hgh, anti, lbord,
        hbord), a the reverse complement of its contig on strand C"""
        g, out, fr = self.g, [], {}
        for c in self.calls:
            ka, kb = (c["ctg1"], c["comp"]), (c["ctg2"], 0)
            for k in (ka, kb):
                if k not in fr:
                    s = g.contig(k[0])
                    fr[k] = ol._framed(3 - s[::-1] if k[1] else s)
            out.append((fr[ka], fr[kb], c["comp"], c["low"], c["hgh"], c["anti"], c["lbord"], c["hbord"]))
        return out

    def reference_keys(self, name):
        """path_key of the reference's Local_Alignment for every call (stored golden)"""
        calls = self.call_args()
        return ol.reference("self_calls/" + name, ol.digest(calls),
                            lambda: ol.ref_local_alignments(calls, self.g.freq))

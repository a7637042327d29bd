"""Crafted inputs of the extension's wave routines: one alignment "tube" per contig pair, seeded by hand, so
that every Local_Alignment call of the path is known in advance and the regimes its wave passes go through
can be steered.  Shared by the CPU pins (test_wave_cases.py, which also records what the reference's
Local_Alignment computes on the oracle's calls) and the GPU test (test_gpu_wave_team.py).

A tube is a core sequence and an edited copy of it, each between flanks of unrelated bases: A = pa + core + sa,
B' = pb + edit(core) + sb.  The edits leave an exact window around the anchor, where three overlapping 40-base
seeds are placed (one chain, one Local_Alignment call).  On strand C the B contig is the reverse complement of
B'.  Seeds are SEED_DT rows in the form the adaptamer merge emits (oracle orc_merge), built by seed_row()."""
import numpy as np

import oracle_lib as ol
from fastga_b200 import formats

PLEN = 40                      # seed length (the k-mer length: the longest seed the merge emits)
SEED_STEP = 23                 # three seeds at +0, +23, +46: 172 anti-diagonals of cover (chain_min 170)
SEED_SPAN = 2 * SEED_STEP + PLEN


def revcomp(a):
    return (3 - a[::-1]).astype(np.uint8)


def seed_row(comp, icont, jcont, x, y, plen, blen):
    """the merge's seed for the match A[x:x+plen] == B'[y:y+plen], B' the B contig (comp 0) or its reverse
    complement (comp 1), icont / jcont contig ranks: a forward A k-mer at post x against a forward B k-mer at
    post y, or against the reverse-strand B k-mer whose post is blen - y (GIXmake: post j+12 of the k-mer
    read backwards from B[j+11])"""
    return (plen, comp, icont, jcont, x, (blen - y) if comp else y)


def seed_match(row, A, B):
    """(x, y, B') of a SEED_DT row against A contig A and B contig B: the match it stands for"""
    plen, comp, _, _, ip, jp = (int(row[f]) for f in ("plen", "comp", "icont", "jcont", "ipost", "jpost"))
    Bp = revcomp(B) if comp else B
    return ip, (len(B) - jp) if comp else jp, Bp


def _edit(rng, seq, sub, indel, maxindel=2):
    """substitutions at rate `sub`, insertions and deletions of 1..maxindel bases at rate `indel` each"""
    out, i, n = [], 0, len(seq)
    r = rng.random(n)
    while i < n:
        if r[i] < indel:
            out.append(rng.integers(0, 4, int(rng.integers(1, maxindel + 1)), dtype=np.uint8))
            out.append(seq[i:i + 1])
        elif r[i] < 2 * indel:
            i += int(rng.integers(1, maxindel + 1))
            continue
        elif r[i] < 2 * indel + sub:
            out.append(np.array([(seq[i] + int(rng.integers(1, 4))) % 4], np.uint8))
        else:
            out.append(seq[i:i + 1])
        i += 1
    return np.concatenate(out) if out else np.zeros(0, np.uint8)


def _runs_copy(rng, lengths, homo=()):
    """(core, copy): exact runs of the given lengths, each followed by one substituted base; runs whose
    index is in `homo` are homopolymers (poly-A and poly-T in turn) flanked by other bases"""
    core, copy = [], []
    prev = -1
    for q, L in enumerate(lengths):
        if q in homo:
            b = 0 if (q // 2) % 2 == 0 else 3
            run = np.full(L, b, np.uint8)
            if prev == b:                                 # the base before a homopolymer is not its base
                core[-1] = copy[-1] = np.array([(b + 1) % 4], np.uint8)
        else:
            run = rng.integers(0, 4, L, dtype=np.uint8)
        a = int(rng.integers(0, 4))
        while a == run[-1]:
            a = int(rng.integers(0, 4))
        c = (a + int(rng.integers(1, 4))) % 4
        while c == run[-1]:
            c = (c + 1) % 4 if (c + 1) % 4 != a else (c + 2) % 4
        core += [run, np.array([a], np.uint8)]
        copy += [run, np.array([c], np.uint8)]
        prev = a
    return np.concatenate(core), np.concatenate(copy)


class Tube:
    """A = pa + left + window + right + sa, B' = pb + left' + window + right' + sb; seeds at the start of
    the window (offset `woff` into it)"""

    def __init__(self, rng, left, left2, right, right2, window=None, pa=0, pb=0, sa=0, sb=0, woff=0, fixed=False,
                 note=""):
        self.window = rng.integers(0, 4, SEED_SPAN + 20, dtype=np.uint8) if window is None else window
        self.left, self.left2, self.right, self.right2 = left, left2, right, right2
        self.flank = [rng.integers(0, 4, n, dtype=np.uint8) for n in (pa, pb, sa, sb)]
        self.woff, self.fixed, self.note = woff, fixed, note
        self.step = SEED_STEP if len(self.window) >= SEED_SPAN else (len(self.window) - PLEN) // 2

    def pad(self, rng, na, nb, front):
        """lengthen the unrelated flanks (front ones when `front`) so that contig lengths are distinct"""
        i = 0 if front else 2
        self.flank[i] = np.concatenate([rng.integers(0, 4, na, dtype=np.uint8), self.flank[i]])
        self.flank[i + 1] = np.concatenate([rng.integers(0, 4, nb, dtype=np.uint8), self.flank[i + 1]])

    @property
    def A(self):
        return np.concatenate([self.flank[0], self.left, self.window, self.right, self.flank[2]])

    @property
    def Bp(self):
        return np.concatenate([self.flank[1], self.left2, self.window, self.right2, self.flank[3]])

    def anchor(self):
        """(x, y) of the first seed"""
        return (len(self.flank[0]) + len(self.left) + self.woff, len(self.flank[1]) + len(self.left2) + self.woff)


def _near_end_tubes(rng, deltas, note):
    """anchors delta bases from the A start, the B start, the A end and the B end: the other contig goes on
    with 2 kbp of unrelated bases; 1.5 kbp of 3 % divergence on the far side"""
    out = []
    for d in deltas:
        for end in ("a0", "b0", "a1", "b1"):
            far = rng.integers(0, 4, 1500, dtype=np.uint8)
            far2 = _edit(rng, far, 0.025, 0.0025)
            near = rng.integers(0, 4, d, dtype=np.uint8)
            if end in ("a0", "b0"):
                t = Tube(rng, near, near.copy(), far, far2, pa=2000 if end == "b0" else 0,
                         pb=2000 if end == "a0" else 0, sa=300, sb=300, note="%s %s %d" % (note, end, d))
            else:
                w = rng.integers(0, 4, SEED_SPAN, dtype=np.uint8)
                t = Tube(rng, far, far2, near, near.copy(), window=w, pa=300, pb=300,
                         sa=2000 if end == "b1" else 0, sb=2000 if end == "a1" else 0,
                         note="%s %s %d" % (note, end, d))
            t.side = end
            out.append(t)
    return out


def _family_tubes(name, rng):
    T = []
    if name == "interior":
        for div in (0.01, 0.03, 0.08):
            halves = []
            for _ in range(2):
                h = rng.integers(0, 4, 15_000, dtype=np.uint8)
                halves += [h, _edit(rng, h, div * 0.85, div * 0.075)]
            T.append(Tube(rng, halves[0], halves[1], halves[2], halves[3], pa=200, pb=200, sa=200, sb=200,
                          note="interior %.0f%%" % (100 * div)))
    elif name == "runs":
        LONG = [31, 32, 33, 47, 63, 64, 65, 95, 96, 97, 127, 128, 129, 500]
        for L in LONG:
            for homo in (False, True):
                sides = []
                for _ in range(2):
                    lens = [int(v) for v in rng.integers(max(1, L // 4), L + 1, max(8, 2500 // L))]
                    lens[1::4] = [L] * len(lens[1::4])
                    if L == 31:
                        lens += list(range(1, 32)) * 2
                        rng.shuffle(lens)
                    h = set(q for q, v in enumerate(lens) if v == L) if homo else ()
                    sides.append(_runs_copy(rng, [min(v, 31) if L == 31 else v for v in lens], h))
                (l1, l2), (r1, r2) = sides
                T.append(Tube(rng, l1, l2, r1, r2, pa=100, pb=100, sa=100, sb=100,
                              note="runs %d%s" % (L, " homopolymer" if homo else "")))
    elif name == "ends":
        T += _near_end_tubes(rng, list(range(0, 131)) + list(range(480, 721, 8)), "ends")
        for sa, sb in ((0, 0), (0, 300), (300, 0)):           # tails: both contigs end together, or one first
            for front in (False, True):
                core = rng.integers(0, 4, 1200, dtype=np.uint8)
                c2 = _edit(rng, core, 0.02, 0.002)
                if front:
                    t = Tube(rng, core, c2, np.zeros(0, np.uint8), np.zeros(0, np.uint8), pa=sa, pb=sb,
                             sa=300, sb=310, note="tail front %d %d" % (sa, sb))
                    t.side = "a0"
                else:
                    t = Tube(rng, np.zeros(0, np.uint8), np.zeros(0, np.uint8), core, c2, pa=300, pb=310,
                             sa=sa, sb=sb, note="tail back %d %d" % (sa, sb))
                    t.side = "a1"
                T.append(t)
        for n in (64, 65, 100, 4095, 4096, 4097, 4160, 8193):  # whole contigs of these lengths, both genomes
            if n < SEED_SPAN + 20:
                w = rng.integers(0, 4, n, dtype=np.uint8)
                t = Tube(rng, np.zeros(0, np.uint8), np.zeros(0, np.uint8), np.zeros(0, np.uint8),
                         np.zeros(0, np.uint8), window=w, woff=(n - SEED_SPAN) // 2 if n >= SEED_SPAN else 0,
                         fixed=True, note="contig %d" % n)
            else:
                m = (n - SEED_SPAN - 20) // 2
                l, r = rng.integers(0, 4, m, dtype=np.uint8), rng.integers(0, 4, n - SEED_SPAN - 20 - m,
                                                                         dtype=np.uint8)
                l2 = l.copy(); r2 = r.copy()
                for s in (l2, r2):                            # substitutions only: B' has A's length
                    q = rng.random(len(s)) < 0.02
                    s[q] = (s[q] + 1) % 4
                t = Tube(rng, l, l2, r, r2, fixed=True, note="contig %d" % n)
            T.append(t)
    elif name in ("bands", "bands_loose"):
        #  a substitution every 45-55 bases keeps the band narrow (a wave advances more than WAVE_LAG): the
        #  widest band is the one the indel opens.  No flanks: the passes end at the contig ends.
        #  the widest band comes out some 11-20 diagonals above L: 0 and 4 stay within 16, 12-15 reach 31
        for L in (0, 4, 8, 12, 13, 14, 15, 16, 17, 24, 28, 30, 31, 32, 40, 120, 250, 300, 400, 500, 700, 1000):
            parts = []
            for side in range(2):
                h = rng.integers(0, 4, 3000, dtype=np.uint8)
                h2 = h.copy()
                q = np.cumsum(rng.integers(45, 56, 3000 // 45))
                q = q[q < len(h)]
                h2[q] = (h2[q] + rng.integers(1, 4, len(q))) % 4
                ins = rng.integers(0, 4, L, dtype=np.uint8)
                cut = 1000 if side == 1 else 2000                 # 1 kbp from the anchor
                if side == 0:                                     # left: L bases missing from B'
                    h2 = np.concatenate([h2[:cut], h2[cut + L:]])
                else:                                             # right: L bases inserted into B'
                    h2 = np.concatenate([h2[:cut], ins, h2[cut:]])
                parts += [h, h2]
            t = Tube(rng, parts[0], parts[1], parts[2], parts[3], note="indel %d" % L)
            t.side = "a1"
            T.append(t)
    else:
        raise KeyError(name)
    return T


#  family -> FastGA flags (param_cases.params) of its run
FLAGS = {"interior": [], "runs": [], "ends": ["-c40"], "bands": [], "bands_loose": ["-i.55"]}
FAMILIES = list(FLAGS)
STRANDS = (0, 1)


class Case:
    """the contigs, seed records and oracle run of one family on one strand"""

    def __init__(self, family, comp):
        import param_cases as pc
        rng = np.random.default_rng(1000 + 10 * FAMILIES.index(family) + comp)
        self.family, self.comp = family, comp
        self.params = pc.params(FLAGS[family])
        self.i_text = next((f[2:] for f in FLAGS[family] if f.startswith("-i")), None)
        tubes = _family_tubes(family, rng)
        # pairwise-distinct contig lengths in each genome: pad flexible tubes' unrelated flanks
        la, lb = set(), set()
        for t in tubes:
            if t.fixed:
                la.add(len(t.A)); lb.add(len(t.Bp))
        for t in tubes:
            if t.fixed:
                continue
            front = getattr(t, "side", "a1") in ("a1", "b1")       # keep the anchored end where it is
            while len(t.A) in la or len(t.Bp) in lb:
                t.pad(rng, 1 if len(t.A) in la else 0, 1 if len(t.Bp) in lb else 0, front)
            la.add(len(t.A)); lb.add(len(t.Bp))
        self.tubes = tubes
        self.A = [t.A for t in tubes]
        self.Bp = [t.Bp for t in tubes]
        self.B = [revcomp(b) if comp else b for b in self.Bp]
        assert len(set(map(len, self.A))) == len(self.A) and len(set(map(len, self.B))) == len(self.B)
        self.gA, self.gB = formats.genome_from_arrays(self.A), formats.genome_from_arrays(self.B)
        self.permA, self.rankA = ol.contig_rank(self.gA.clen)
        self.permB, self.rankB = ol.contig_rank(self.gB.clen)
        self.layout = ol.seed_layout(self.gA, self.gB)
        rows = []
        for i, t in enumerate(tubes):
            x, y = t.anchor()
            for k in range(3):
                rows.append(seed_row(comp, self.rankA[i], self.rankB[i], x + k * t.step, y + k * t.step,
                                     PLEN, len(self.B[i])))
        self.seeds = np.array(rows, dtype=ol.SEED_DT)
        self.recs = ol.seed_records(self.seeds, self.layout, sort=True)
        self._run = None

    @property
    def freq(self):
        return self.gA.freq

    @property
    def ave_corr(self):
        return 1.0 - self.params.get("align_rate", 0.3)

    def search_kw(self):
        return {k: v for k, v in self.params.items() if k in ("chain_break", "chain_min", "align_min", "align_rate")}

    def run(self):
        """ol.search_calls on the crafted records: (records, pool, nhit, calls, passes)"""
        if self._run is None:
            self._run = ol.search_calls(self.recs, self.layout, self.gA, self.gB, self.permA, self.permB,
                                        self.freq, **self.search_kw())
        return self._run

    def seam_jobs(self):
        """the logged calls as Local_Alignment jobs (A contig, B contig, comp, low, hgh, anti, lbord, hbord)"""
        calls = self.run()[3]
        return np.array([(c["ctg1"], c["ctg2"], c["comp"], c["low"], c["hgh"], c["anti"], c["lbord"], c["hbord"])
                         for c in calls], dtype=np.int32).reshape(-1, 8)

    def reference(self):
        """path_key of the reference's Local_Alignment for every logged call"""
        import param_cases as pc
        calls = pc.seam_calls(self.A, self.B, self.seam_jobs())
        return ol.reference("wave_team/%s_%s" % (self.family, "NC"[self.comp]),
                            ol.digest(calls, self.freq, self.ave_corr),
                            lambda: ol.ref_local_alignments(calls, self.freq, self.ave_corr))


_cases = {}


def case(family, comp):
    if (family, comp) not in _cases:
        _cases[(family, comp)] = Case(family, comp)
    return _cases[(family, comp)]


# ------------------------------------------------------------------------------------------------
#  what the oracle's passes must show on each family (both strands unless a row says otherwise)
# ------------------------------------------------------------------------------------------------

BAND_BINS = {"band<=16": (0, 16), "band17-30": (17, 30), "band31": (31, 31), "band32-251": (32, 251),
             "band>=252": (252, 1 << 30)}


def call_band(passes, c):
    """the widest band of a call's passes"""
    return int(passes["maxband"][c["pass0"]:c["pass0"] + c["npass"]].max())


def regimes_reached(calls, passes):
    """the set of regime names the passes reach"""
    got = set()
    for c in calls:
        if c["npass"] == 0:
            continue
        w = call_band(passes, c)
        got |= {k for k, (lo, hi) in BAND_BINS.items() if lo <= w <= hi}
    for p in passes:
        d = "fwd" if p["s"] > 0 else "rev"
        got.add("snake==%d" % p["maxsnake"])
        if p["aend"]:
            got.add("aend_" + d)
        if p["bend"]:
            got.add("bend_" + d)
        if p["endempty"]:
            got.add("endempty_" + d)
        if p["maxhop"] > 256:
            got.add("hop>256")
        if p["narrowspan"] > 8192:
            got.add("long_narrow_" + d)
        for name, v in (("da0", p["da0"]), ("da1", p["da1"]), ("db0", p["db0"]), ("db1", p["db1"])):
            if v <= 130:
                got.add("near_" + name)
            elif 500 <= v <= 800:
                got.add("lookahead_" + name)
    return got


#  family -> regimes its passes must reach on each strand.  endempty_*: a wave that meets a contig end
#  keeps no diagonal within WAVE_LAG after the end clip -- the one way to the device's "wave did not
#  advance" bail-out (front_run: m == 0), since besta itself never stalls (oracle wave(); the test
#  asserts it).  Every band >= 252 call (the wide-band kernel) also hops over more than 64 cells, the
#  window of that kernel's pebble walk (WIDE_HOP); no crafted band stays over 256 diagonals for a whole
#  trace-point interval, so no pass hops over 256 cells, the window of the shared-memory kernel.
WIDE_HOP = 64
REGIMES = {
    "interior": {"long_narrow_fwd", "long_narrow_rev"},
    "runs": {"snake==31", "snake==32", "snake==33", "snake==63", "snake==64", "snake==65", "snake==500"},
    "ends": {"aend_fwd", "aend_rev", "bend_fwd", "bend_rev", "endempty_fwd", "endempty_rev", "near_da0", "near_da1", "near_db0", "near_db1",
             "lookahead_da0", "lookahead_da1", "lookahead_db0", "lookahead_db1"},
    "bands": {"band<=16", "band17-30", "band32-251", "endempty_fwd", "endempty_rev"},
    "bands_loose": {"band<=16", "band17-30", "band31", "band32-251", "band>=252"},
}

"""Edge-case inputs shared by the GPU parity tests and the CPU oracle-pin tests: ragged and tiny
contigs, unrelated genomes (empty result), identical and reverse-complemented copies, tandem
repeats (frequency cutoff, wide bands), many small contigs.  Each case returns
(A contigs, B contigs, reference threads, check(alignments, hits)); reference_run(name) is what the
reference computed on it."""
import os
import tempfile

import numpy as np

from fastga_b200 import synth


def _distinct(contigs):
    seen, out = set(), []
    for c in contigs:
        while len(c) in seen:
            c = c[:-1]
        seen.add(len(c))
        out.append(c)
    return out


def ragged():
    rng = np.random.default_rng(51)
    core = rng.integers(0, 4, 150_003, dtype=np.uint8)
    A = _distinct([core[:70_001], core[70_001:], rng.integers(0, 4, 39, dtype=np.uint8),
                   rng.integers(0, 4, 11, dtype=np.uint8), rng.integers(0, 4, 41, dtype=np.uint8)])
    mut = synth._small_mutations(rng, core, 0.04)
    B = _distinct([mut[:33_333], mut[33_333:], rng.integers(0, 4, 13, dtype=np.uint8)])
    return A, B, 4, lambda al, hits: len(al) > 0


def unrelated():
    rng = np.random.default_rng(52)
    A = _distinct([rng.integers(0, 4, 300_000, dtype=np.uint8), rng.integers(0, 4, 200_000, dtype=np.uint8)])
    B = _distinct([rng.integers(0, 4, 400_000, dtype=np.uint8)])
    def check(al, hits):
        assert len(al) == 0 and hits == 0
    return A, B, 4, check


def identical_and_revcomp():
    rng = np.random.default_rng(53)
    a1 = rng.integers(0, 4, 400_000, dtype=np.uint8)
    a2 = rng.integers(0, 4, 250_001, dtype=np.uint8)
    B = _distinct([a1.copy()[:399_990], (3 - a2[::-1]).astype(np.uint8)])
    def check(al, hits):
        assert {int(x) for x in al.fields[:, 0]} == {0, 1}
    return [a1, a2], B, 4, check


def tandem_repeats():
    rng = np.random.default_rng(54)
    parts = []
    while sum(len(p) for p in parts) < 600_000:
        parts.append(rng.integers(0, 4, int(rng.integers(20_000, 60_000)), dtype=np.uint8))
        unit = rng.integers(0, 4, int(rng.integers(20, 400)), dtype=np.uint8)
        parts.append(np.concatenate([synth._small_mutations(rng, unit, 0.02)
                                     for _ in range(int(rng.integers(20, 120)))]))
    a = np.concatenate(parts)[:600_000]
    B = [synth.diverged_copy(rng, a, 0.04, sv_every=80_000)]
    return [a], B, 4, lambda al, hits: len(al) > 0


def many_small_contigs():
    rng = np.random.default_rng(55)
    base = rng.integers(0, 4, 1_200_000, dtype=np.uint8)
    cuts = np.sort(rng.choice(np.arange(2_000, 1_198_000), 119, replace=False))
    A = _distinct(list(np.split(base, cuts)))
    mut = synth._small_mutations(rng, base, 0.08)
    cuts2 = np.sort(rng.choice(np.arange(2_000, len(mut) - 2_000), 60, replace=False))
    B = _distinct(list(np.split(mut, cuts2)))
    return A, B, 8, lambda al, hits: len(al) > 50


#  Width boundaries of the packed records.  The seed key has 2*bitlen(amx+bmx) + 7 + J + I bits
#  (J, I = bit widths of the B / A contig ranks); past 64 bits its upper fields move into the second
#  word.  A .ktab contig field is 2 bytes once 2*ncontig > 256, a position field 4 bytes once a contig
#  is longer than 2^24, and the contig rank is a 15-bit field.  REGIMES below states what each case
#  reaches; tests/test_host_logic.py checks that it does.

def _wide_pair(seed, na, nb, long_len=700_000):
    """one ~700 kbp contig per genome (longest A + longest B in [2^20, 2^21)) plus 2-8 kbp contigs;
    B's short contigs are diverged copies of A contigs drawn from every length rank"""
    rng = np.random.default_rng(seed)
    a0 = rng.integers(0, 4, long_len, dtype=np.uint8)
    A = _distinct([a0] + [rng.integers(0, 4, int(rng.integers(2_000, 8_000)), dtype=np.uint8)
                          for _ in range(na - 1)])
    src = rng.choice(np.arange(1, na), nb - 1, replace=False)
    B = _distinct([synth.diverged_copy(rng, a0, 0.05, sv_every=60_000)] +
                  [synth.diverged_copy(rng, A[int(k)], 0.05, sv_every=0) for k in src])
    return A, B


def seed_key_64():
    A, B = _wide_pair(71, 200, 100)
    return A, B, 8, lambda al, hits: len(al) > 50


def seed_key_65():
    A, B = _wide_pair(72, 200, 129)
    return A, B, 8, lambda al, hits: len(al) > 50


def icont_straddles():
    A, B = _wide_pair(73, 300, 200)
    return A, B, 8, lambda al, hits: len(al) > 50 and int(al.fields[:, 1].max()) > 255


LONG = (1 << 24) + 300_000


def _long_genomes(rng):
    """one contig of 2^24 + 300 kbp per genome; homology only in a forward window that straddles
    2^24 in both and a reverse-complemented window past 2^24 in A that straddles 2^24 of B's
    complement (C-strand records count B positions on the complement), the rest unrelated, which
    keeps the oracle cheap; plus two short unrelated contigs each"""
    a = rng.integers(0, 4, LONG, dtype=np.uint8)
    fa, ra, rb = (1 << 24) - 40_000, (1 << 24) + 120_000, 270_000
    inv = synth._revcomp(synth._small_mutations(rng, a[ra:ra + 60_000], 0.04))
    parts = [rng.integers(0, 4, rb, dtype=np.uint8), inv, rng.integers(0, 4, fa - rb - len(inv), dtype=np.uint8),
             synth._small_mutations(rng, a[fa:fa + 80_000], 0.04)]
    n = sum(len(p) for p in parts)
    b = np.concatenate(parts + [rng.integers(0, 4, LONG - 17 - n, dtype=np.uint8)])
    A = [a, rng.integers(0, 4, 50_000, dtype=np.uint8), rng.integers(0, 4, 30_001, dtype=np.uint8)]
    B = [b, rng.integers(0, 4, 40_000, dtype=np.uint8), rng.integers(0, 4, 20_001, dtype=np.uint8)]
    return A, B


def _past_2_24_on_both_strands(al, hits):
    f = al.fields
    big = (f[:, 5] > (1 << 24)) & (f[:, 6] > (1 << 24))
    assert big.any() and set(int(c) for c in f[big, 0]) == {0, 1}


def long_contigs():
    A, B = _long_genomes(np.random.default_rng(74))
    return A, B, 4, _past_2_24_on_both_strands


def long_and_many():
    rng = np.random.default_rng(75)
    A, B = _long_genomes(rng)
    # 150 short B contigs, every third a diverged copy of a piece of A's long contig past 2^24
    for k in range(150):
        n = int(rng.integers(2_000, 6_000))
        if k % 3 == 0:
            s = int(rng.integers((1 << 24) + 200_000, LONG - n))
            B.append(synth._small_mutations(rng, A[0][s:s + n], 0.04))
        else:
            B.append(rng.integers(0, 4, n, dtype=np.uint8))
    B = _distinct(B)

    def check(al, hits):
        _past_2_24_on_both_strands(al, hits)
        assert int(al.fields[:, 2].max()) > 127
    return A, B, 4, check


MAX_CONTIGS = 0x7fff


def max_contigs():
    """32767 A contigs: 770 of 1-2.9 kbp cut from a 1.5 Mbp sequence that B (200 contigs) is a
    diverged copy of, and 31997 unrelated 60-400 bp fillers.  Filler lengths repeat, so their ranks
    depend on the sort's tie order; every filler is shorter than every homologous contig, so the
    homologous ranks do not, and fillers carry no alignments."""
    rng = np.random.default_rng(76)
    lens = rng.choice(np.arange(1_000, 2_900), 770, replace=False)
    base = rng.integers(0, 4, int(lens.sum()), dtype=np.uint8)
    hom = np.split(base, np.cumsum(lens)[:-1])
    fill = [rng.integers(0, 4, int(n), dtype=np.uint8) for n in rng.integers(60, 401, MAX_CONTIGS - len(hom))]
    A = hom + fill
    order = rng.permutation(len(A))
    A = [A[i] for i in order]
    mut = synth.diverged_copy(rng, base, 0.05, sv_every=50_000, inversions=False)
    cuts = np.sort(rng.choice(np.arange(1_000, len(mut) - 1_000), 199, replace=False))
    B = _distinct(list(np.split(mut, cuts)))
    return A, B, 8, lambda al, hits: len(al) > 100


def chain_islands():
    """one contig pair of 200 homologous islands of 100-130 bp between unrelated spacers of 1100-1500 bp,
    equal in A and B (longer than chain_break / 2, so every island is a chain of its own).  An island of B
    is its A island with every 18th base substituted: no indels, so all its seeds lie on one diagonal
    inside one 64-wide band, and a substitution every 18 bases leaves about 15 seeds per chain.  So one
    band-pair triple holds 180-odd chains in two chunks of chain detection, far more than the 48 a chunk
    records, and is scanned in the extension kernel instead.  Eight more pairs, diverged copies with
    indels, hold few chains each in band pairs of thousands of seeds."""
    rng = np.random.default_rng(77)
    a, b = [], []
    for _ in range(200):
        isl = rng.integers(0, 4, int(rng.integers(100, 131)), dtype=np.uint8)
        sub = np.arange(len(isl)) % 18 == 17
        mut = isl.copy()
        mut[sub] = (mut[sub] + rng.integers(1, 4, int(sub.sum()))) % 4
        n = int(rng.integers(1_100, 1_501))
        a += [isl, rng.integers(0, 4, n, dtype=np.uint8)]
        b += [mut, rng.integers(0, 4, n, dtype=np.uint8)]
    A = [np.concatenate(a)] + [rng.integers(0, 4, int(rng.integers(40_000, 60_000)), dtype=np.uint8) for _ in range(8)]
    B = [np.concatenate(b)] + [synth.diverged_copy(rng, c, 0.05, sv_every=0, inversions=False) for c in A[1:]]
    return _distinct(A), _distinct(B), 4, lambda al, hits: hits >= 180 and len(al) >= 180


def wave_regimes():
    """the crafted wave tubes of wave_cases.py, the `ends` family on strand N and the `runs` family on strand
    C, as one genome pair, aligned from natural seeds: anchors near every contig end, tails, short and
    4 kbp-boundary contigs, exact runs of 31..500 bases and homopolymer runs"""
    import wave_cases as wc
    e, r = wc.case("ends", 0), wc.case("runs", 1)
    return _distinct(e.A + r.A), _distinct(e.B + r.B), 4, lambda al, hits: len(al) >= 600


CASES = {"ragged": ragged, "unrelated": unrelated, "identical_and_revcomp": identical_and_revcomp,
         "tandem_repeats": tandem_repeats, "many_small_contigs": many_small_contigs,
         "seed_key_64": seed_key_64, "seed_key_65": seed_key_65, "icont_straddles": icont_straddles,
         "long_contigs": long_contigs, "long_and_many": long_and_many, "max_contigs": max_contigs,
         "chain_islands": chain_islands, "wave_regimes": wave_regimes}

#  what each width case must reach: seed key bits, (post_bytes, cont_bytes) of A and of B, and for
#  the long cases the least longest-contig length; chunk_overflow: a chunk of chain detection holds more
#  chains than it records (tests/test_gpu_chains.py checks it)
REGIMES = {"seed_key_64": dict(key=64, gixA=(3, 2), gixB=(3, 1)),
           "seed_key_65": dict(key=65, gixA=(3, 2), gixB=(3, 2)),
           "icont_straddles": dict(key=66, gixA=(3, 2), gixB=(3, 2)),
           "long_contigs": dict(key=63, gixA=(4, 1), gixB=(4, 1), maxlen=1 << 24),
           "long_and_many": dict(key=69, gixA=(4, 1), gixB=(4, 2), maxlen=1 << 24),
           "max_contigs": dict(key=62, gixA=(2, 2), gixB=(2, 2), ncontigA=MAX_CONTIGS),
           # a chunk of chain detection with more than 48 chains: its triple has no hit list
           "chain_islands": dict(key=55, gixA=(3, 1), gixB=(3, 1), chunk_overflow=True)}


def reference_run(name):
    """the reference's -v counters and canonical records on case `name` (oracle_lib.reference)"""
    import oracle_lib as ol
    from fastga_b200 import formats
    A, B, threads, _ = CASES[name]()

    def run():
        with tempfile.TemporaryDirectory() as wd:
            formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", 1))
            formats.write_fasta(os.path.join(wd, "B.fasta"), synth.scaffolds_of(B, "sb", 1))
            return ol.ref_alignments(wd, "A", "B", threads)
    return ol.reference("edge/" + name, ol.digest(A, B, threads), run)

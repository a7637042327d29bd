"""Inputs of the tests that run the alignment path at non-default FastGA parameters (-c -s -l -i -f) and on
genomes of skewed base composition, shared by the CPU pins (test_params.py, which also records what the
reference computed on them) and the GPU tests (test_gpu_params.py, which only read those records).

A case is (flags, pair generator): the flags are FastGA's own command-line options, and params() turns them
into the library's keyword arguments the way FastGA's option parser does (FastGA.c:4493-4548)."""
import os
import tempfile

import numpy as np

from fastga_b200 import synth
from edge_cases import _distinct, tandem_repeats

THREADS = 8


def params(flags):
    """FastGA options -> keyword arguments of lib.fastga / ol.oracle_pipeline.  -c and -s are doubled
    (anti-diagonal space); -i is parsed with strtod and stored as ALIGN_RATE = 1.-i, so the rate is
    1.0 - float(text), never the decimal literal of 1-i (-i.8 gives mscore 199, not 200)."""
    p = {}
    for f in flags:
        opt, val = f[1], f[2:]
        if opt == "c":
            p["chain_min"] = 2 * int(val)
        elif opt == "s":
            p["chain_break"] = 2 * int(val)
        elif opt == "l":
            p["align_min"] = int(val)
        elif opt == "f":
            p["freq"] = int(val)
        elif opt == "i":
            p["align_rate"] = 1.0 - float(val)
        else:
            raise ValueError(f)
    return p


def ave_corr(i_text):
    """the ave_corr New_Align_Spec sees for -i<i_text>: 1.-ALIGN_RATE with ALIGN_RATE = 1.-strtod(i_text)"""
    return 1.0 - (1.0 - float(i_text))


def composed_contigs(rng, total_bp, ncontig, at):
    """ncontig pairwise-distinct lengths summing to ~total_bp, bases drawn with P(A) = P(T) = at/2"""
    w = rng.uniform(0.5, 1.5, ncontig)
    lens = np.maximum((w / w.sum() * total_bp).astype(np.int64), 1000) + np.arange(ncontig)
    p = np.array([at / 2, (1 - at) / 2, (1 - at) / 2, at / 2])
    return [rng.choice(4, int(n), p=p).astype(np.uint8) for n in lens]


def composed_pair(seed, total_bp, ncontig, div, sv_every, at=0.5):
    """(A contigs, B contigs): B contig i is a diverged copy (synth.diverged_copy) of A contig i, emitted in
    a shuffled order; lengths pairwise distinct in each genome"""
    rng = np.random.default_rng(seed)
    A = composed_contigs(rng, total_bp, ncontig, at)
    B = [synth.diverged_copy(rng, a, div, sv_every) for a in A]
    B = [B[i] for i in rng.permutation(ncontig)]
    return _distinct(A), _distinct(B)


def _tandem():
    A, B, _, _ = tandem_repeats()
    return A, B


#  name -> (FastGA flags, pair generator, what the case reaches)
CASES = {
    "strict": (["-i.9", "-l500"], lambda: composed_pair(71, 1_500_000, 3, 0.05, 60_000),
               "ave_path 54: many hits rejected by rate and length"),
    "loose": (["-i.55", "-l50"], lambda: composed_pair(72, 350_000, 3, 0.18, 30_000),
              "ave_path 33: wide bands, the +.05 acceptance slack (slow on the CPU: kept small)"),
    "short_chains": (["-c20", "-s100"], lambda: composed_pair(73, 1_000_000, 3, 0.08, 50_000),
                     "many chain breaks and hits per triple (a dozen chains at most in one chunk of chain "
                     "detection: the 48-chain overflow is edge_cases.chain_islands)"),
    "long_break": (["-c500", "-s20000"], lambda: composed_pair(74, 1_500_000, 3, 0.05, 20_000),
                   "chains bridging SV gaps, 13 seeds before a triple is scanned"),
    "freq3": (["-f3"], _tandem, "frequency cutoff 3 on tandem repeats"),
    "freq60": (["-f60"], _tandem, "frequency cutoff 60 on tandem repeats"),
    "at_rich": ([], lambda: composed_pair(75, 1_500_000, 3, 0.05, 60_000, at=0.70),
                "A+T = 0.70: bias index 5"),
    "gc_rich": (["-i.8"], lambda: composed_pair(76, 1_500_000, 3, 0.05, 60_000, at=0.15),
                "A+T = 0.15: the 80/20 cap (bias 3) with a non-default rate"),
}


def case(name):
    """(flags, A contigs, B contigs) of case `name`"""
    flags, make, _ = CASES[name]
    A, B = make()
    return flags, A, B


def reference_run(name, A, B):
    """the reference's -v counters and canonical records on case `name` (A, B from case(name)):
    FastGA -v -k -T8 <flags> A B"""
    import oracle_lib as ol
    from fastga_b200 import formats
    flags = CASES[name][0]

    def run():
        with tempfile.TemporaryDirectory() as wd:
            formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(A, "sa", 1))
            formats.write_fasta(os.path.join(wd, "B.fasta"), synth.scaffolds_of(B, "sb", 1))
            return ol.ref_alignments(wd, "A", "B", THREADS, extra=flags)
    return ol.reference("params/" + name, ol.digest(A, B, THREADS, flags), run)


#  SELF mode: the `dup` genome of test_oracle_pin._self_genomes at these flags
SELF_NAME = "dup"
SELF_FLAGS = ["-c40", "-s400", "-i.85"]
SELF_THREADS = 4


def self_reference_run(genome):
    import oracle_lib as ol
    from fastga_b200 import formats

    def run():
        with tempfile.TemporaryDirectory() as wd:
            formats.write_fasta(os.path.join(wd, "A.fasta"), synth.scaffolds_of(genome, "sa", 1))
            return ol.ref_alignments(wd, "A", None, SELF_THREADS, extra=SELF_FLAGS)
    return ol.reference("params/self_" + SELF_NAME, ol.digest(genome, SELF_THREADS, SELF_FLAGS), run)


# ------------------------------------------------------------------------------------------------
#  batched Local_Alignment (the align.h seam) at other identities and on a skewed composition
# ------------------------------------------------------------------------------------------------

def seam_jobs(seed, borders, at=None):
    """contigs A, diverged copies B and 300 Local_Alignment jobs (A contig, B contig, comp, low, hgh, anti,
    lbord, hbord) around the copies' diagonals.  at=None draws bases uniformly (the draws of the original
    seam test); else with P(A) = P(T) = at/2."""
    rng = np.random.default_rng(seed)
    ncont = 6
    if at is None:
        A = [rng.integers(0, 4, int(rng.integers(3000, 40000)), dtype=np.uint8) for _ in range(ncont)]
    else:
        p = np.array([at / 2, (1 - at) / 2, (1 - at) / 2, at / 2])
        A = [rng.choice(4, int(rng.integers(3000, 40000)), p=p).astype(np.uint8) for _ in range(ncont)]
    B = []
    for a in A:
        rate = float(rng.choice([0.02, 0.05, 0.1, 0.15]))
        b = synth.diverged_copy(rng, a, rate, sv_every=0, inversions=False)      # small mutations only
        B.append(np.concatenate([rng.integers(0, 4, int(rng.integers(0, 300)), dtype=np.uint8), b]))
    jobs = []
    for _ in range(300):
        i = int(rng.integers(0, ncont))
        comp = int(rng.random() < 0.4)
        la, lb = len(A[i]), len(B[i])
        x = int(rng.integers(100, la - 100))
        y = int(np.clip(x + (lb - la) + int(rng.integers(-60, 60)), 50, lb - 50))
        if comp:                       # the strand-C call sees reverse-complemented A: any diagonal will do
            y = int(rng.integers(50, lb - 50))
        d, anti = x - y, x + y
        low, hgh = d - int(rng.integers(0, 70)), d + int(rng.integers(0, 70))
        lbd = hbd = -1
        if borders:
            lbd = int(rng.integers(0, 40)) if rng.random() < 0.7 else -1
            hbd = int(rng.integers(0, 40)) if rng.random() < 0.7 else -1
        jobs.append((i, i, comp, low, hgh, anti, lbd, hbd))
    return A, B, np.array(jobs, dtype=np.int32)


def seam_calls(A, B, jobs):
    """the jobs as reference Local_Alignment calls (framed a, framed b, comp, low, hgh, anti, lbord, hbord)"""
    import oracle_lib as ol
    fA = [ol._framed(a) for a in A]
    fAC = [ol._framed(3 - a[::-1]) for a in A]
    fB = [ol._framed(b) for b in B]
    return [((fAC[i] if comp else fA[i]), fB[j], comp, low, hgh, anti, lbd, hbd)
            for (i, j, comp, low, hgh, anti, lbd, hbd) in jobs.tolist()]


#  name -> (-i text, A+T of the A contigs or None for uniform)
SEAM_CASES = {"i0.55": ("0.55", None), "i0.8": ("0.8", None), "i0.95": ("0.95", None), "at0.3": ("0.7", 0.3)}


def seam_case(name):
    """(A, B, jobs, calls, A's frequency vector, -i text) of a seam case; borders on, seed 43"""
    from fastga_b200 import formats
    i_text, at = SEAM_CASES[name]
    A, B, jobs = seam_jobs(43, True, at)
    return A, B, jobs, seam_calls(A, B, jobs), formats.genome_from_arrays(A).freq, i_text


def seam_reference(name, calls, freq, i_text):
    """path_key of the reference's Local_Alignment for every call of seam case `name`"""
    import oracle_lib as ol
    ac = ave_corr(i_text)
    return ol.reference("local_alignment/seam_" + name, ol.digest(calls, freq, ac),
                        lambda: ol.ref_local_alignments(calls, freq, ac))

"""-m gpu: k-mer tables from one syncmer scan, sorted along two routes, in one process.  By default the sort
starts from the scan's layout, the records in runs by the first digit of the k-mer partition; with
FGB_KSORT_PARTITION=1 it ignores that layout and runs every partition pass in Onesweep.  The table, the
prefix index and the sampler histogram must be byte-identical; the LCP bytes are computed from the table by
the same kernel.  Every table is also pinned to the oracle's: a both-strand table and its prefix index
equal the oracle's, a forward-only table the oracle's forward-strand entries, a range table the oracle's
entries whose 12-base prefix lies in the range.  The sharded path's scan (lib.kmers_scan) is pinned to the
built tables."""
import numpy as np
import pytest
import torch

import bench
import oracle_lib as ol
from fastga_b200 import formats, lib, synth

pytestmark = pytest.mark.gpu

BK_CAP = 4096      # records a CTA of the bucket sort holds; larger bins take the oversized-bin path
REV = np.uint64(1 << 47)        # strand bit of a record's lo word (top bit of the contig field)

_oracle = {}


def oracle_table(genome, crank):
    """the oracle's both-strand table and prefix index of a genome; the last two genomes' are kept (the genome
    with them, so that its id is not reused)"""
    key = id(genome)
    if key not in _oracle:
        if len(_oracle) >= 2:
            del _oracle[next(iter(_oracle))]
        _oracle[key] = (genome, ol.gix_build(genome, crank))
    return _oracle[key][1]


def _build(dg, kind, plo, phi):
    if kind == "both":
        x = lib.DeviceGix.build(dg)
    elif kind == "forward":
        x = lib.DeviceGix.build_forward(dg)
    else:
        x = lib.DeviceGix.build_range(dg, plo, phi)
    try:
        tab, pstart, buck = x.download()
        return x.n, tab, pstart, buck
    finally:
        x.close()


def assert_matches_oracle(genome, crank, kind, plo, phi, n, tab, pstart):
    want, wstart = oracle_table(genome, crank)
    if kind == "both":
        assert np.array_equal(pstart, wstart)
    elif kind == "forward":
        want = want[(want[:, 0] & REV) == 0]
    else:
        prefix = want[:, 1] >> np.uint64(40)
        want = want[(prefix >= plo) & (prefix < phi)]
    assert n == len(want)
    assert tab.tobytes() == want.tobytes()


def assert_paths_agree(monkeypatch, genome, kinds=("both", "forward"), plo=0, phi=1 << 24):
    dg = lib.DeviceGenome(genome)
    out = []
    for kind in kinds:
        monkeypatch.delenv("FGB_KSORT_PARTITION", raising=False)
        got = _build(dg, kind, plo, phi)
        monkeypatch.setenv("FGB_KSORT_PARTITION", "1")
        want = _build(dg, kind, plo, phi)
        monkeypatch.delenv("FGB_KSORT_PARTITION")
        assert got[0] == want[0] == len(got[1])
        for g, w in zip(got[1:], want[1:]):
            assert g.tobytes() == w.tobytes()
        assert_matches_oracle(genome, dg.crank, kind, plo, phi, *got[:3])
        out.append(got)
    return out


@pytest.mark.parametrize("kind", ["both", "forward"])
def test_small_pair(small_pair, monkeypatch, kind):
    for g in small_pair:
        (n, _, _, _), = assert_paths_agree(monkeypatch, g, (kind,))
        assert n > 100_000


def test_heavy_repeats(monkeypatch):
    rng = np.random.default_rng(77)
    unit = rng.integers(0, 4, 37, dtype=np.uint8)
    contigs = [rng.integers(0, 4, 300_000, dtype=np.uint8), np.tile(unit, 8000),
               np.zeros(50_000, dtype=np.uint8), rng.integers(0, 4, 150_001, dtype=np.uint8)]
    assert_paths_agree(monkeypatch, formats.genome_from_arrays(contigs))


def test_bench_generator_few_mbp(monkeypatch):
    A, B = synth.make_pair(bench.SEED, 3_000_000, bench.NCONTIG, bench.DIV, sv_every=bench.SV_EVERY)
    for g in (A, B):
        (n, tab, _, _), _ = assert_paths_agree(monkeypatch, formats.genome_from_arrays(g))
        assert n > 1_000_000
        assert (np.diff(tab[:, 1].astype(np.float64)) >= 0).all()


def test_tandem_repeats(monkeypatch):
    """crowded sub-bins send bucket-sort groups down the LSD path, crowded bins down the oversized-bin path"""
    rng = np.random.default_rng(5)
    contigs = [np.tile(rng.integers(0, 4, k, dtype=np.uint8), 200_000 // k) for k in (3, 12, 37, 101)]
    contigs.append(rng.integers(0, 4, 100_000, dtype=np.uint8))
    assert_paths_agree(monkeypatch, formats.genome_from_arrays(contigs))


def test_contigs_shorter_than_12_and_40_bases(monkeypatch):
    """contigs below 12 bases are not scanned; below 40 they are scanned but give no entry (a forward
    entry needs 40 bases after it, a reverse one 28 before and 12 after)"""
    rng = np.random.default_rng(12)
    lens = [1, 5, 11, 12, 13, 27, 28, 29, 39, 40, 41, 63, 64, 65, 4095, 4096, 4097, 20_000]
    assert_paths_agree(monkeypatch, formats.genome_from_arrays([rng.integers(0, 4, n, dtype=np.uint8)
                                                                for n in lens]))
    short = formats.genome_from_arrays([rng.integers(0, 4, n, dtype=np.uint8) for n in (3, 11, 20, 39)])
    for n, _, pstart, _ in assert_paths_agree(monkeypatch, short):
        assert n == 0 and not pstart.any()


def test_short_contigs(monkeypatch):
    rng = np.random.default_rng(6)
    lens = [1, 11, 12, 13, 27, 28, 39, 40, 41, 1023, 1024, 1025, 4096, 4097, 9000]
    assert_paths_agree(monkeypatch, formats.genome_from_arrays([rng.integers(0, 4, n, dtype=np.uint8)
                                                                for n in lens]))
    only_short = formats.genome_from_arrays([rng.integers(0, 4, n, dtype=np.uint8) for n in (5, 11, 30, 39)])
    for n, _, pstart, _ in assert_paths_agree(monkeypatch, only_short):
        assert n == 0 and not pstart.any()


def test_skewed_composition(monkeypatch):
    """mostly A: one first digit holds most records, so most tiles store one long run"""
    rng = np.random.default_rng(7)
    skew = rng.choice(4, size=600_000, p=[0.85, 0.05, 0.05, 0.05]).astype(np.uint8)
    gc = rng.choice(4, size=300_000, p=[0.05, 0.45, 0.45, 0.05]).astype(np.uint8)
    assert_paths_agree(monkeypatch, formats.genome_from_arrays([skew, gc]))


def test_prefix_ranges(small_pair, monkeypatch):
    g = small_pair[1]
    cuts = [0, 3, 1 << 16, (1 << 22) + 99, (1 << 23) + 1, 1 << 24]
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        assert_paths_agree(monkeypatch, g, ("range",), lo, hi)
    (n, _, _, _), = assert_paths_agree(monkeypatch, g, ("range",), 77777, 77777)
    assert n == 0


def test_uneven_prefix_shares(small_pair, monkeypatch):
    g = small_pair[1]
    cuts = [0, 1, 1 << 21, (1 << 23) + 12345, (1 << 23) + 12346, (3 << 22) + 7, 1 << 24]
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        assert_paths_agree(monkeypatch, g, ("range",), lo, hi)
    (n, _, _, _), = assert_paths_agree(monkeypatch, g, ("range",), 5000, 5000)
    assert n == 0


@pytest.mark.parametrize("target", ["24", "4", "1"])
def test_finer_bins(small_pair, monkeypatch, target):
    """a lower bin target stands for a larger genome: the partition then sorts more prefix bits, in more
    Onesweep passes and with first digits of other widths"""
    monkeypatch.setenv("FGB_KSORT_BIN_TARGET", target)
    assert_paths_agree(monkeypatch, small_pair[0])
    assert_paths_agree(monkeypatch, small_pair[1], ("range",), 1 << 20, 5 << 21)


@pytest.mark.parametrize("target", ["8", "1"])
def test_more_than_65536_bins(small_pair, monkeypatch, target):
    monkeypatch.setenv("FGB_KSORT_BIN_TARGET", target)
    g = small_pair[1]
    assert_paths_agree(monkeypatch, g, ("both",))
    assert_paths_agree(monkeypatch, small_pair[0], ("forward",))
    for lo, hi in ((0, (1 << 23) + 5), ((1 << 23) + 5, 1 << 24)):
        assert_paths_agree(monkeypatch, g, ("range",), lo, hi)


def test_one_oversized_bin_among_many_empty_bins(monkeypatch):
    """a short random contig leaves most of the 65536 bins empty; a poly-A run puts all of its forward
    entries into the first bin, far above what one CTA of the bucket sort holds"""
    rng = np.random.default_rng(4)
    g = formats.genome_from_arrays([rng.integers(0, 4, 3000, dtype=np.uint8), np.zeros(3 * BK_CAP, dtype=np.uint8)])
    (n, tab, _, _), = assert_paths_agree(monkeypatch, g, ("forward",))
    prefix = tab[:, 1] >> np.uint64(40)
    bins, counts = np.unique(prefix >> np.uint64(8), return_counts=True)
    assert counts.max() > BK_CAP and len(bins) < 65536 // 8
    assert_paths_agree(monkeypatch, g, ("both",))


class _DeviceRecords:
    """n 16-byte device records as a CUDA array, for torch to copy to the host"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n, 2), "typestr": "<i8", "data": (ptr, False),
                                          "strides": None, "version": 3}


def scanned_records(dg, mask, fwd):
    ptr, n = lib.kmers_scan(dg, mask, fwd)
    try:
        recs = torch.as_tensor(_DeviceRecords(ptr, n), device="cuda").cpu().numpy().view(np.uint64)
    finally:
        lib.device_free(ptr)
    return recs[np.lexsort((recs[:, 0], recs[:, 1]))]


@pytest.mark.parametrize("fwd", [False, True])
def test_kmers_scan(small_pair, fwd):
    """the sharded path's scan gives the records of the built table; with a mask, those of the selected
    contigs (a record carries its contig's rank, bits 32-46 of lo)"""
    for g in small_pair:
        dg = lib.DeviceGenome(g)
        x = lib.DeviceGix.build_forward(dg) if fwd else lib.DeviceGix.build(dg)
        tab = x.download(want_index=False)[0]
        x.close()
        assert np.array_equal(scanned_records(dg, np.ones(g.ncontig, dtype=np.uint8), fwd), tab)
        mask = (np.arange(g.ncontig) % 2 == 0).astype(np.uint8)
        assert 0 < mask.sum() < g.ncontig
        rank = (tab[:, 0] >> np.uint64(32)) & np.uint64(0x7fff)
        want = tab[np.isin(rank, dg.crank[mask != 0].astype(np.uint64))]
        assert 0 < len(want) < len(tab)
        assert np.array_equal(scanned_records(dg, mask, fwd), want)

"""-m gpu: k-mer tables whose records the scan scatters straight into their prefix bins, against the same
tables laid out by the Onesweep partition passes (FGB_KSORT_PARTITION=1), in one process.  The table,
the prefix index, the sampler histogram and the record count must be byte-identical."""
import numpy as np
import pytest

from fastga_b200 import formats, lib

pytestmark = pytest.mark.gpu

BK_CAP = 4096      # records a CTA of the bucket sort holds; larger bins take the oversized-bin path


def _build(dg, kind, plo, phi):
    if kind == "both":
        x = lib.DeviceGix.build(dg)
    elif kind == "forward":
        x = lib.DeviceGix.build_forward(dg)
    else:
        x = lib.DeviceGix.build_range(dg, plo, phi)
    tab, pstart, buck = x.download()
    return x.n, tab, pstart, buck


def assert_paths_agree(monkeypatch, genome, kind="both", plo=0, phi=1 << 24):
    dg = lib.DeviceGenome(genome)
    monkeypatch.delenv("FGB_KSORT_PARTITION", raising=False)
    got = _build(dg, kind, plo, phi)
    monkeypatch.setenv("FGB_KSORT_PARTITION", "1")
    want = _build(dg, kind, plo, phi)
    monkeypatch.delenv("FGB_KSORT_PARTITION")
    assert got[0] == want[0] == len(got[1])
    for g, w in zip(got[1:], want[1:]):
        assert g.tobytes() == w.tobytes()
    return got


@pytest.mark.parametrize("kind", ["both", "forward"])
def test_small_pair(small_pair, monkeypatch, kind):
    for g in small_pair:
        n, _, _, _ = assert_paths_agree(monkeypatch, g, kind)
        assert n > 100_000


def test_heavy_repeats(monkeypatch):
    rng = np.random.default_rng(77)
    unit = rng.integers(0, 4, 37, dtype=np.uint8)
    contigs = [rng.integers(0, 4, 300_000, dtype=np.uint8), np.tile(unit, 8000),
               np.zeros(50_000, dtype=np.uint8), rng.integers(0, 4, 150_001, dtype=np.uint8)]
    g = formats.genome_from_arrays(contigs)
    for kind in ("both", "forward"):
        assert_paths_agree(monkeypatch, g, kind)


def test_contigs_shorter_than_12_and_40_bases(monkeypatch):
    """contigs below 12 bases are not scanned; below 40 they are scanned but give no entry (a forward
    entry needs 40 bases after it, a reverse one 28 before and 12 after)"""
    rng = np.random.default_rng(12)
    lens = [1, 5, 11, 12, 13, 27, 28, 29, 39, 40, 41, 63, 64, 65, 4095, 4096, 4097, 20_000]
    g = formats.genome_from_arrays([rng.integers(0, 4, n, dtype=np.uint8) for n in lens])
    for kind in ("both", "forward"):
        assert_paths_agree(monkeypatch, g, kind)
    short = formats.genome_from_arrays([rng.integers(0, 4, n, dtype=np.uint8) for n in (3, 11, 20, 39)])
    for kind in ("both", "forward"):
        n, _, pstart, _ = assert_paths_agree(monkeypatch, short, kind)
        assert n == 0 and not pstart.any()


def test_uneven_prefix_shares(small_pair, monkeypatch):
    g = small_pair[1]
    cuts = [0, 1, 1 << 21, (1 << 23) + 12345, (1 << 23) + 12346, (3 << 22) + 7, 1 << 24]
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        assert_paths_agree(monkeypatch, g, "range", lo, hi)
    assert_paths_agree(monkeypatch, g, "range", 5000, 5000)


@pytest.mark.parametrize("target", ["8", "1"])
def test_more_than_65536_bins(small_pair, monkeypatch, target):
    monkeypatch.setenv("FGB_KSORT_BIN_TARGET", target)
    g = small_pair[1]
    assert_paths_agree(monkeypatch, g, "both")
    assert_paths_agree(monkeypatch, small_pair[0], "forward")
    for lo, hi in ((0, (1 << 23) + 5), ((1 << 23) + 5, 1 << 24)):
        assert_paths_agree(monkeypatch, g, "range", lo, hi)


def test_one_oversized_bin_among_many_empty_bins(monkeypatch):
    """a short random contig leaves most of the 65536 bins empty; a poly-A run puts all of its forward
    entries into the first bin, far above what one CTA of the bucket sort holds"""
    rng = np.random.default_rng(4)
    g = formats.genome_from_arrays([rng.integers(0, 4, 3000, dtype=np.uint8), np.zeros(3 * BK_CAP, dtype=np.uint8)])
    n, tab, _, _ = assert_paths_agree(monkeypatch, g, "forward")
    prefix = tab[:, 1] >> np.uint64(40)
    bins, counts = np.unique(prefix >> np.uint64(8), return_counts=True)
    assert counts.max() > BK_CAP and len(bins) < 65536 // 8
    assert_paths_agree(monkeypatch, g, "both")

"""-m gpu: k-mer tables whose scan stores its records in runs by the first digit of the k-mer partition,
against the same tables built from records packed tile after tile and laid out by Onesweep partition
passes alone (FGB_KSORT_PARTITION=1), in one process.  The table, the prefix index and the sampler
histogram must be byte-identical; the LCP bytes are computed from the table by the same kernel."""
import numpy as np
import pytest

import bench
from fastga_b200 import formats, lib, synth

pytestmark = pytest.mark.gpu


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
        out.append(got)
    return out


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


@pytest.mark.parametrize("target", ["24", "4", "1"])
def test_finer_bins(small_pair, monkeypatch, target):
    """a lower bin target stands for a larger genome: the partition then sorts more prefix bits, in more
    Onesweep passes and with first digits of other widths"""
    monkeypatch.setenv("FGB_KSORT_BIN_TARGET", target)
    assert_paths_agree(monkeypatch, small_pair[0])
    assert_paths_agree(monkeypatch, small_pair[1], ("range",), 1 << 20, 5 << 21)

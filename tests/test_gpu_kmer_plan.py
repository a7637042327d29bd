"""k-mer tables planned on the device: the fine-bin starts come from a lower-bound search over the partitioned
records and the bucket-sort groups from a planning kernel, so a table build waits on the host only for the
count pass's total and, at its end, for the plan's count of bins too large for a CTA.  The tables are pinned to
the oracle and to FGB_KSORT_PARTITION=1 by test_gpu_kmer_build; this file counts the waits, covers the routes
that file does not (an empty range, the sharded table from records), and checks the restated packing rule
(kmer_sort_cases.plan_groups) on random bin sizes."""
import numpy as np
import pytest

from fastga_b200 import formats, lib

from kmer_sort_cases import BK_SPAN, plan_groups
from test_gpu_kmer_build import BK_CAP, _DeviceRecords, assert_matches_oracle, assert_paths_agree, scanned_records

@pytest.mark.parametrize("seed", range(6))
def test_packing_keeps_bins_whole(seed):
    rng = np.random.default_rng(seed)
    nbins = int(rng.integers(1, 3000))
    sizes = rng.choice([0, 1, 700, 1500, 2100, BK_CAP, BK_CAP + 1, 3 * BK_CAP], nbins,
                       p=[0.3, 0.1, 0.2, 0.2, 0.1, 0.05, 0.03, 0.02])
    bins = np.concatenate([[0], np.cumsum(sizes)])
    groups, over = plan_groups(bins)
    covered = np.zeros(int(bins[-1]), dtype=np.int32)
    for gs, gc, gp in groups:
        assert 0 < gc <= BK_CAP
        assert gs == bins[gp]
        end = int(np.searchsorted(bins, gs + gc, side="left"))
        assert bins[end] == gs + gc                    # ends on a bin boundary
        assert end - gp <= BK_SPAN and gp // BK_SPAN == (end - 1) // BK_SPAN
        covered[gs:gs + gc] += 1
    for os_, oc in over:
        assert oc > BK_CAP
        covered[os_:os_ + oc] += 1
    assert (covered == 1).all()
    assert len(groups) <= nbins


@pytest.mark.gpu
def test_table_builds_wait_twice(small_pair):
    gA, gB = small_pair
    dA, dB = lib.DeviceGenome(gA), lib.DeviceGenome(gB)
    w0 = lib.host_waits()
    x = lib.DeviceGix.build(dB)
    assert lib.host_waits() - w0 == 2
    x.close()
    _, stats = lib.fastga(gA, gB)
    assert stats["gix_waits"] == 2
    _, stats = lib.fastga_self(gA)
    assert stats["gix_waits"] == 2


@pytest.mark.gpu
def test_oversized_bins_wait_more(monkeypatch):
    rng = np.random.default_rng(4)
    g = formats.genome_from_arrays([rng.integers(0, 4, 3000, dtype=np.uint8), np.zeros(3 * BK_CAP, dtype=np.uint8)])
    dg = lib.DeviceGenome(g)
    w0 = lib.host_waits()
    x = lib.DeviceGix.build(dg)
    assert lib.host_waits() - w0 > 2
    x.close()
    monkeypatch.setenv("FGB_KSORT_BIN_TARGET", "1")
    assert_paths_agree(monkeypatch, g, ("both", "forward"))


@pytest.mark.gpu
def test_empty_range(small_pair):
    dg = lib.DeviceGenome(small_pair[0])
    for plo, phi in ((5000, 5000), (0, 0)):
        x = lib.DeviceGix.build_range(dg, plo, phi)
        try:
            tab, pstart, _ = x.download()
            assert x.n == 0 and len(tab) == 0
        finally:
            x.close()


@pytest.mark.gpu
@pytest.mark.parametrize("target", [None, "1"])
@pytest.mark.parametrize("fwd", [False, True])
def test_table_from_records(small_pair, monkeypatch, fwd, target):
    """the sharded route: scanned records in any order, sorted by fgb_gix_from_records, over the whole range and
    over one share of it"""
    import torch
    if target:
        monkeypatch.setenv("FGB_KSORT_BIN_TARGET", target)
    g = small_pair[1]
    dg = lib.DeviceGenome(g)
    mask = np.ones(g.ncontig, dtype=np.uint8)
    ptr, n = lib.kmers_scan(dg, mask, fwd)
    try:
        recs = torch.as_tensor(_DeviceRecords(ptr, n), device="cuda")
        for plo, phi in ((0, 1 << 24), (1 << 22, 3 << 22)):
            pre = (recs[:, 1] >> 40) & 0xffffff
            share = recs[(pre >= plo) & (pre < phi)].contiguous()
            x = lib.gix_from_records(share.data_ptr(), share.shape[0], plo, phi, fwd, 4, 2, g.ncontig)
            try:
                nx = x.n
                tab, pstart, _ = x.download()
            finally:
                x.close()
            rows = share.cpu().numpy().view(np.uint64).copy().view([("lo", "<u8"), ("hi", "<u8")]).reshape(-1)
            want = np.sort(rows, order=("hi", "lo")).view(np.uint64).reshape(-1, 2)
            assert tab.tobytes() == want.tobytes()
            if plo == 0 and not fwd:
                assert_matches_oracle(g, dg.crank, "both", 0, 1 << 24, nx, tab, pstart)
    finally:
        lib.device_free(ptr)

"""-m gpu: the crafted inputs of kmer_sort_cases.py through the k-mer table sort and the syncmer scan.

Record cases go through fgb_gix_from_records (records in any order, no first digit): the table must equal
numpy's sort by (hi, lo) byte for byte, the prefix index a searchsorted over the prefixes (built again after
the bins too large for the bucket sort), and the build must wait on the host once when the restated plan has
no such bins and more often when it has some (fgb_kmer_sort_oversized waits on its own).

Genome cases are built along both routes (the scan's first-digit layout and FGB_KSORT_PARTITION=1) and pinned
to the oracle; their sampler histogram must equal the restated one, and for a whole-range case the unsorted
records of lib.kmers_scan must lie in runs by the restated first digit, in digit order, tile by tile within a
run, each (digit, tile) run holding exactly that tile's oracle records (their order inside a run is the emit
pass's atomic order and is not compared)."""
import numpy as np
import pytest
import torch

import kmer_sort_cases as kc
import oracle_lib as ol
from fastga_b200 import lib
from test_gpu_kmer_build import _DeviceRecords, assert_paths_agree, oracle_table

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _target(monkeypatch, target):
    if target is None:
        monkeypatch.delenv("FGB_KSORT_BIN_TARGET", raising=False)
    else:
        monkeypatch.setenv("FGB_KSORT_BIN_TARGET", str(target))


@pytest.mark.parametrize("name", kc.RECORD_NAMES)
def test_record_case(name, monkeypatch):
    c = kc.record_case(name)
    _target(monkeypatch, c.target)
    P = kc.record_plan(c.records, c.plo, c.phi, c.target, _sms())
    if name.startswith("cta_loop"):
        assert len(P["groups"]) > 3 * P["grid"]
    n = len(c.records)
    d = torch.from_numpy(c.records.view(np.int64)).cuda()
    torch.cuda.synchronize()
    w0 = lib.host_waits()
    x = lib.gix_from_records(d.data_ptr() if n else 0, n, c.plo, c.phi, False, 4, 2, 1 << 15)
    waits = lib.host_waits() - w0
    try:
        assert x.n == n
        tab, pstart, _ = x.download()
    finally:
        x.close()
    want = P["tab"]
    assert tab.tobytes() == want.tobytes()
    assert np.array_equal(pstart, kc.prefix_index(want))
    if P["over"]:
        assert waits > 1, waits
    else:
        assert waits == 1, waits


def _scan_records(dg, fwd):
    ptr, n = lib.kmers_scan(dg, np.ones(dg.genome.ncontig, dtype=np.uint8), fwd)
    try:
        return torch.as_tensor(_DeviceRecords(ptr, n), device="cuda").cpu().numpy().view(np.uint64).copy()
    finally:
        lib.device_free(ptr)


def _by_key(key, recs):
    o = np.lexsort((recs[:, 0], recs[:, 1], key))
    return key[o], recs[o]


@pytest.mark.parametrize("name", kc.GENOME_NAMES)
def test_genome_case(name, monkeypatch):
    c = kc.genome_case(name)
    _target(monkeypatch, c.target)
    g = c.genome
    dg = lib.DeviceGenome(g)
    rank = ol.contig_rank(g.clen)[1]
    assert np.array_equal(dg.crank, rank)
    if c.full_range:
        # the scan's layout first: the sort's first partition pass takes its digit histogram from the count pass,
        # so it relies on the emit pass writing exactly the records that pass counted
        want = kc.case_table(c, oracle_table(g, dg.crank)[0])
        fsh, dbits, _ = kc.scan_layout(c, len(want))
        got = _scan_records(dg, c.kind == "forward")
        key = kc.scan_key(c, got, rank, fsh, dbits)
        assert (np.diff(key) >= 0).all(), "records out of their (digit, tile) run"
        k1, r1 = _by_key(key, got)
        k2, r2 = _by_key(kc.scan_key(c, want, rank, fsh, dbits), want)
        assert np.array_equal(k1, k2)
        assert r1.tobytes() == r2.tobytes()
    (n, tab, pstart, buck), = assert_paths_agree(monkeypatch, g, (c.kind,), c.plo, c.phi)
    assert np.array_equal(buck, kc.buck1024(c.contigs))

"""-m gpu: every call gives back the device blocks it took from the block cache -- on success once its
handles are closed, and on an error return reached after it has allocated."""
import ctypes as C

import numpy as np
import pytest

from fastga_b200 import formats, lib, load_library
from param_cases import seam_jobs

pytestmark = pytest.mark.gpu


def live():
    return lib.device_live_bytes()


def device_alloc(nbytes):
    L = load_library()
    p = C.c_void_p()
    assert L.fgb_device_alloc(nbytes, C.byref(p), None) == 0
    return p.value


class _Range(C.Structure):
    _fields_ = [("beg", C.c_int), ("end", C.c_int), ("off", C.c_longlong)]


def seam_genomes(seed=41):
    A, B, jobs = seam_jobs(seed, False)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    return gA, gB, np.ascontiguousarray(jobs, dtype=np.int32).reshape(-1, 8)


def test_whole_path_calls_leave_no_live_blocks(small_pair):
    gA, gB = small_pair
    base = live()
    alns, _ = lib.fastga(gA, gB)
    assert len(alns) > 0
    assert live() == base
    alns, _ = lib.fastga_self(gA)
    assert live() == base
    dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
    held = live()
    assert held > base
    alns, _ = lib.align_resident(dA, dB, gA.freq)
    assert len(alns) > 0
    assert live() == held
    dA.close()
    dB.close()
    assert live() == base


def test_sharded_building_blocks_leave_no_live_blocks(small_pair):
    gA, gB = small_pair
    dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
    base = live()
    tables = []
    for dg, fwd in ((dA, True), (dB, False)):
        g = dg.genome
        ptr, n = lib.kmers_scan(dg, np.ones(g.ncontig, dtype=np.uint8), fwd)
        grouped = device_alloc(16 * max(n, 1))
        bounds = lib.records_group_by_owner(ptr, n, np.zeros(256, dtype=np.int32), 1, grouped)
        assert bounds[-1] == n
        lib.device_free(ptr)
        pb, cb = formats.gix_bytes(g)
        tables.append(lib.gix_from_records(grouped, n, 0, 1 << 24, fwd, pb, cb, g.ncontig))
        lib.device_free(grouped)
    xA, xB = tables
    amx, bmx = int(gA.clen.max()), int(gB.clen.max())
    sptr, ns, bits, sumlen, _ = lib.seeds_merge(xA, xB, amx, bmx)
    xA.close()
    xB.close()
    assert ns > 0
    grouped = device_alloc(16 * ns)
    bounds = lib.seeds_group_by_owner(sptr, ns, bits, np.zeros(gA.ncontig, dtype=np.int32), 1, grouped)
    assert bounds[-1] == ns
    lib.device_free(sptr)
    S = lib.seeds_from_records(grouped, ns, bits, amx, bmx, sumlen)
    lib.device_free(grouped)
    ov = lib.DeviceOverlaps.extend(S, dA, dB, gA.freq)
    alns = lib.filter_overlaps(ov.h, dA.perm, dB.perm, bits[2], bits[3])
    ov.close()
    S.close()
    assert len(alns) > 0
    assert live() == base
    dA.close()
    dB.close()


def test_stage_calls_leave_no_live_blocks(small_pair):
    gA, gB, jobs = seam_genomes()
    dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
    base = live()
    paths, _, _ = lib.local_alignments(dA, dB, jobs, gA.freq)
    assert (paths[:, 6] == 0).all()
    assert live() == base
    dA.close()
    dB.close()

    sA, sB = small_pair
    dA, dB = lib.DeviceGenome(sA, want_revcomp=True), lib.DeviceGenome(sB, want_revcomp=True)
    alns, _ = lib.align_resident(dA, dB, sA.freq)
    base = live()
    soff, _, _ = lib.compute_trace_pts(dA, dB, alns)
    assert len(soff) == len(alns) + 1
    assert live() == base
    dA.close()
    dB.close()

    rng = np.random.default_rng(3)
    base = live()
    lib.sort128_host(rng.integers(0, 1 << 63, size=(100_003, 2), dtype=np.uint64), 0, 16)
    assert live() == base

    L = load_library()
    rsize, ksize, beg, end = 15, 10, 3, 40
    counts = rng.integers(0, 3000, end - beg)
    n = int(counts.sum())
    arr = np.concatenate([rng.integers(0, 256, n * rsize, dtype=np.uint8), np.zeros(16, np.uint8)])
    part = np.zeros(1024, dtype=np.int64)
    part[beg:end] = counts * rsize
    L.fgb_msd_sort(arr.ctypes.data, n, rsize, ksize, part.ctypes.data, beg, end, 4)
    assert live() == base

    rsize, nparts, nthreads = 9, 37, 8
    counts = rng.integers(0, 5000, nparts)
    n = int(counts.sum())
    arr = rng.integers(0, 256, n * rsize, dtype=np.uint8)
    part = (counts * rsize).astype(np.int64)
    ranges = (_Range * nthreads)()
    assert L.fgb_rmsd_sort(arr.ctypes.data, n, rsize, rsize, nparts, part.ctypes.data, nthreads, ranges) > 0
    assert live() == base


def test_ktab_export_and_import_leave_no_live_blocks(small_pair):
    g = small_pair[0]
    dg = lib.DeviceGenome(g)
    base = live()
    gx = lib.DeviceGix.build(dg)
    _, pstart, _ = gx.download()
    ent = gx.export_ktab(np.zeros(1, dtype=np.int64))
    gf = formats.GixFile()
    gf.entries, gf.n, gf.post_bytes, gf.cont_bytes = ent, gx.n, gx.post_bytes, gx.cont_bytes
    gf.index, gf.ncontig = pstart[1:].astype(np.int64), g.ncontig
    imp = lib.DeviceGix.import_ktab(gf)
    assert imp.n == gx.n
    imp.close()
    gx.close()
    assert live() == base
    dg.close()


def test_seed_sort_refusal_releases_its_blocks():
    """records with hi bits under a key of <= 64 bits: FGB_ERR_ARG after the sort has run"""
    import torch
    rng = np.random.default_rng(9)
    recs = np.zeros((20_000, 2), dtype=np.uint64)
    recs[:, 0] = rng.integers(0, 1 << 63, size=len(recs), dtype=np.uint64)
    recs[12_345, 1] = 1
    d = torch.from_numpy(recs.view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    L = load_library()
    bits = (C.c_int * 4)(25, 19, 3, 3)                  # key of 63 bits
    h = C.c_void_p()
    base = live()
    rc = L.fgb_seeds_from_records(C.c_void_p(d.data_ptr()), len(recs), bits, 1, 1, 0, C.byref(h), None)
    assert rc == -2 and not h.value
    assert live() == base


def test_local_alignments_overflow_releases_its_blocks(monkeypatch):
    """traces_cap = 0 on calls that produce traces: FGB_ERR_OVERFLOW once the records are back; and
    FGB_ERR_OVERFLOW from a record buffer too small for the records (FGB_EXTEND_OUT_SLACK), with at
    least the trace bytes needed"""
    gA, gB, jobs = seam_genomes()
    dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
    tables, ave = lib.align_spec(0.7, gA.freq)
    L = load_library()

    def call(jobs):
        n = jobs.shape[0]
        paths = np.zeros((n, 7), dtype=np.int32)
        toff = np.zeros(n, dtype=np.int64)
        traces = np.zeros(1, dtype=np.uint8)
        used = C.c_longlong()
        base = live()
        rc = L.fgb_local_alignments(dA.h, dB.h, n, jobs.ctypes.data, tables.ctypes.data, ave, 100,
                                    paths.ctypes.data, toff.ctypes.data, traces.ctypes.data, 0, C.byref(used), None)
        assert live() == base
        return rc, used.value

    rc, used = call(jobs)
    assert rc == -4 and used > 0
    # records of 40 + tlen (padded to 8) bytes over the 256 a job is given, more than 64 in all
    paths, _, _ = lib.local_alignments(dA, dB, jobs, gA.freq)
    big = np.ascontiguousarray(jobs[paths[:, 5] >= 300])
    assert len(big) > 0
    monkeypatch.setenv("FGB_EXTEND_OUT_SLACK", "64")
    rc, used = call(big)
    assert rc == -4 and used >= int(paths[paths[:, 5] >= 300, 5].sum())
    dA.close()
    dB.close()

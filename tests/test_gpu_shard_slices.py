"""-m gpu: the data flow of shard.align_sharded for every rank of a world W, in one process and without
collectives: each exchange is the concatenation of every source rank's group for the destination, in
source-rank order, as all_to_all_single delivers it.  Each step is checked against the single-GPU stage it
stands in for:
  * slice tables: rank r's table, built by gix_from_records from what the k-mer scans of all ranks sent
    it, equals the oracle's table restricted to r's prefix range (A: its forward-strand entries), with the
    prefix index of that restriction; B's also equals DeviceGix.build_range over the whole genome;
  * seeds: seeds_merge per slice gives the oracle's merge of the restricted tables, and the union over the
    slices gives the count, the sum of seed lengths and the records of DeviceSeeds.find on whole tables;
  * per-rank seeds: after seeds_group_by_owner and seeds_from_records, rank r's sorted seeds are the whole
    sorted seed set, in its order, filtered to the A-contig ranks r owns.
A pair with fewer contigs than ranks and a two-letter alphabet leaves ranks without contigs to scan and
slices without records."""
import numpy as np
import pytest
import torch

import oracle_lib as ol
from edge_cases import _distinct
from fastga_b200 import formats, lib, shard, synth
from multi_worker import seed_icont

pytestmark = pytest.mark.gpu

REV = np.uint64(1 << 47)        # strand bit of a k-mer record's lo word


class _DeviceRecords:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n, 2), "typestr": "<i8", "data": (ptr, False),
                                          "strides": None, "version": 3}


def records_at(ptr, n):
    if n == 0:
        return np.zeros((0, 2), dtype=np.uint64)
    return torch.as_tensor(_DeviceRecords(ptr, n), device="cuda").cpu().numpy().view(np.uint64)


def pstart_of(T):
    pre = (T[:, 1] >> np.uint64(40)).astype(np.int64)
    return np.searchsorted(pre, np.arange((1 << 24) + 1)).astype(np.int64)


def restrict(T, ps, plo, phi):
    """rows of a sorted table T (prefix index ps) whose prefix lies in [plo, phi), and their prefix index"""
    a, b = ps[plo], ps[phi]
    return T[a:b], np.clip(ps - a, 0, b - a).astype(np.uint32)


def exchange(parts, world):
    """parts[s] = (grouped rows of source rank s, bounds): what each rank receives, in source-rank order"""
    out = []
    for r in range(world):
        got = [g[int(b[r]):int(b[r + 1])] for g, b in parts if b[r + 1] > b[r]]
        out.append(torch.cat(got) if got else torch.empty((0, 2), dtype=torch.int64, device="cuda"))
    return out


def sharded_flow(gA, gB, world):
    dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
    ownA, ownB = shard.owner_of_contigs(gA.clen, world), shard.owner_of_contigs(gB.clen, world)
    cuts = shard.top_byte_cuts(world)
    owner256 = np.zeros(256, dtype=np.int32)
    for r in range(world):
        owner256[cuts[r]:cuts[r + 1]] = r
    recv = []
    for dg, own, fwd in ((dA, ownA, True), (dB, ownB, False)):
        parts = []
        for s in range(world):
            ptr, n = lib.kmers_scan(dg, (own == s).astype(np.uint8), fwd)
            grouped = torch.empty((max(n, 1), 2), dtype=torch.int64, device="cuda")
            try:
                bounds = lib.records_group_by_owner(ptr, n, owner256, world, grouped.data_ptr())
            finally:
                lib.device_free(ptr)
            assert bounds[-1] == n
            parts.append((grouped, bounds))
        recv.append(exchange(parts, world))
    return dA, dB, ownA, recv


def prefix_cuts(world):
    """rank r owns the k-mers whose top byte lies in [ceil(256 r / W), ceil(256 (r+1) / W)): the first
    256 mod W ranks one byte more than the others (86/85/85 at W = 3)"""
    return [-(-256 * r // world) for r in range(world + 1)]


def check_flow(gA, gB, world):
    dA, dB, ownA, (recvA, recvB) = sharded_flow(gA, gB, world)
    cuts = prefix_cuts(world)
    tA, _ = ol.gix_build(gA, dA.crank)
    tA = tA[(tA[:, 0] & REV) == 0]
    tB, _ = ol.gix_build(gB, dB.crank)
    psA, psB = pstart_of(tA), pstart_of(tB)
    amx, bmx = int(gA.clen.max()), int(gB.clen.max())
    (pbA, cbA), (pbB, cbB) = formats.gix_bytes(gA), formats.gix_bytes(gB)
    assert sum(len(r) for r in recvA) == len(tA) and sum(len(r) for r in recvB) == len(tB)

    xa, xb = lib.DeviceGix.build_forward(dA), lib.DeviceGix.build(dB)
    whole = lib.DeviceSeeds.find(xa, xb, amx, bmx)
    xa.close()
    xb.close()
    wrec, wn, wsum, layout = whole.download(), whole.n, whole.sumlen, whole.layout
    whole.close()

    seeds, nseeds, sumlen = [], 0, 0
    for r in range(world):
        plo, phi = cuts[r] << 16, cuts[r + 1] << 16
        want = []
        for recv, T, ps, fwd, pb, cb, g in ((recvA[r], tA, psA, True, pbA, cbA, gA),
                                            (recvB[r], tB, psB, False, pbB, cbB, gB)):
            x = lib.gix_from_records(recv.data_ptr() if len(recv) else 0, len(recv), plo, phi, fwd, pb, cb,
                                     g.ncontig)
            tab, pstart, _ = x.download()
            wt, wps = restrict(T, ps, plo, phi)
            assert x.n == len(wt) == len(recv), (r, fwd)
            assert tab.tobytes() == wt.tobytes(), (r, fwd)
            assert np.array_equal(pstart, wps), (r, fwd)
            if not fwd:
                y = lib.DeviceGix.build_range(dB, plo, phi)
                ytab, ypstart, _ = y.download()
                y.close()
                assert tab.tobytes() == ytab.tobytes() and np.array_equal(pstart, ypstart), r
            want.append((x, wt, wps))
        (x1, t1, _), (x2, t2, ps2) = want
        sptr, ns, bits, sl, n1m = lib.seeds_merge(x1, x2, amx, bmx)
        x1.close()
        x2.close()
        oseeds, osum = ol.merge(t1, t2, ps2)
        assert (ns, sl, n1m) == (len(oseeds), osum, len(t1)), r
        assert tuple(bits) == layout, r
        seeds.append((sptr, ns))
        nseeds += ns
        sumlen += sl
    assert (nseeds, sumlen) == (wn, wsum)

    union = np.concatenate([records_at(p, n) for p, n in seeds])
    assert np.array_equal(union[np.lexsort((union[:, 0], union[:, 1]))], wrec[np.lexsort((wrec[:, 0], wrec[:, 1]))])

    own_by_rank = ownA[dA.perm]
    parts = []
    for sptr, ns in seeds:
        grouped = torch.empty((max(ns, 1), 2), dtype=torch.int64, device="cuda")
        try:
            bounds = lib.seeds_group_by_owner(sptr, ns, layout, own_by_rank, world, grouped.data_ptr())
        finally:
            if sptr:
                lib.device_free(sptr)
        parts.append((grouped, bounds))
    wowner = own_by_rank[seed_icont(wrec, 12 + layout[0] + layout[1] + layout[2], layout[3])]
    for r, recv in enumerate(exchange(parts, world)):
        S = lib.seeds_from_records(recv.data_ptr() if len(recv) else 0, len(recv), layout, amx, bmx)
        got = S.download()
        S.close()
        assert np.array_equal(got, wrec[wowner == r]), r
    return recvA, recvB


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8, 64])
def test_small_pair_slices_and_seeds(small_pair, world):
    recvA, recvB = check_flow(*small_pair, world)
    assert all(len(r) > 0 for r in recvA + recvB)


def test_fewer_contigs_than_ranks_and_empty_slices():
    """two contigs per genome over the bases 0 and 1, at world 8: ranks 2-7 scan nothing.  A forward k-mer
    then has a top byte of 2-bit digits 0 and 1, a reverse one of digits 2 and 3; of the eight 32-value
    slices, A's records reach ranks 0 and 2 only, B's ranks 0, 2, 5 and 7, so ranks 1, 3, 4 and 6 build
    and merge empty slices of both genomes"""
    A, B = synth.make_pair(23, 400_000, 2, 0.04, sv_every=50_000)
    A, B = _distinct([a & 1 for a in A]), _distinct([b & 1 for b in B])
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    recvA, recvB = check_flow(gA, gB, 8)
    assert [r for r in range(8) if len(recvA[r])] == [0, 2]
    assert [r for r in range(8) if len(recvB[r])] == [0, 2, 5, 7]

"""torchrun worker for tests/test_gpu_multi.py: the k-mer-space sharded path (shard.align_sharded:
every rank scans its contigs, k-mer records and seeds are exchanged with all-to-alls, every rank
extends the seeds of its A-contigs); rank 0 gathers the record streams and checks the union against
a single-GPU run of the whole pair.  FGB_MULTI_BACKEND: nccl (default; one GPU per rank) or gloo
(ranks may share a GPU).  FGB_MULTI_PAIR: "few_contigs" (three contigs per genome, fewer than the
ranks of a world of 8, and a B contig with two exact copies of one A segment) or a case of
tests/edge_cases.py in place of the default pair.  Rank 0 also checks the gathered records in their
gathered order against the single-GPU run's .1aln order.

Every rank holds both genomes, so a seed routed to the wrong rank would still be extended correctly
and the union of the records would not show it: every rank also decodes the icont field of each seed
it received and checks that it owns that A-contig rank."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np          # noqa: E402
import torch                # noqa: E402
import torch.distributed as dist   # noqa: E402
from fastga_b200 import formats, lib, shard, synth   # noqa: E402


def seed_icont(recs, p_ic, ic_bits):
    """the icont field (A-contig rank) of (n,2) uint64 seed records [lo, hi], at bit p_ic of the 128"""
    lo, hi = recs[:, 0], recs[:, 1]
    if p_ic >= 64:
        v = hi >> np.uint64(p_ic - 64)
    else:
        v = (lo >> np.uint64(p_ic)) | (hi << np.uint64(64 - p_ic))
    return (v & np.uint64((1 << ic_bits) - 1)).astype(np.int64)


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    backend = os.environ.get("FGB_MULTI_BACKEND", "nccl")
    local = int(os.environ.get("LOCAL_RANK", rank)) % torch.cuda.device_count()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if backend == "nccl":
        dist.init_process_group("nccl", device_id=dev)
    else:
        dist.init_process_group(backend)
    case = os.environ.get("FGB_MULTI_PAIR")
    if case == "few_contigs":
        A, B = synth.make_pair(78, 3_000_000, 3, 0.05, sv_every=80_000)
        # two exact copies of one A segment in a B contig, each between 100 bases that differ from A's
        # flanks at every position: two alignments with the same A interval, tied on (aread, abpos, bread,
        # comp), whose order only the discovery order sets
        import edge_cases
        seg = np.concatenate([3 - A[0][99_900:100_000], A[0][100_000:130_000], 3 - A[0][130_000:130_100]])
        B[1] = np.concatenate([B[1][:50_000], seg, B[1][50_000:60_000], seg, B[1][60_000:]])
        B = edge_cases._distinct(B)
    elif case:
        import edge_cases
        A, B, _, _ = edge_cases.CASES[case]()
    else:
        A, B = synth.make_pair(77, 6_000_000, 6, 0.05, sv_every=80_000)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    dA, dB = lib.DeviceGenome(gA, want_revcomp=True), lib.DeviceGenome(gB)
    received = []
    alns, st = shard.align_sharded(dA, dB, gA.freq, dist, dev,
                                   on_seeds=lambda recv, bits: received.append((recv.cpu().numpy(), bits)))
    recs, bits = received[0]
    ic = seed_icont(recs.view(np.uint64), 12 + bits[0] + bits[1] + bits[2], bits[3])
    own_by_rank = shard.owner_of_contigs(gA.clen, world)[dA.perm]
    if not (own_by_rank[ic] == rank).all():
        print("OWNER_MISMATCH rank=%d icont=%s" % (rank, np.unique(ic[own_by_rank[ic] != rank])[:10].tolist()),
              flush=True)
        raise AssertionError("rank %d received seeds of A-contig ranks it does not own" % rank)
    print("RANK_OK rank=%d contigs=%d seeds=%d records=%d" % (rank, int((shard.owner_of_contigs(gA.clen, world)
                                                                        == rank).sum()), len(recs), len(alns)),
          flush=True)
    tot = torch.tensor([st["nkmers1_fwd"], st["nkmers2"], st["nseeds_merged"], st["nseeds"], st["nhits"]],
                       dtype=torch.int64, device=dev)
    dist.all_reduce(tot)
    maxic = torch.tensor([int(ic.max()) if len(ic) else -1], dtype=torch.int64, device=dev)
    dist.all_reduce(maxic, op=dist.ReduceOp.MAX)
    merged = shard.gather_alignments(alns, None, dist, dev)
    if rank == 0:
        whole, ws = lib.align_resident(dA, dB, gA.freq)
        t = [int(v) for v in tot.tolist()]
        assert t[0] == ws["nkmers1_fwd"] and t[1] == ws["nkmers2"], (t, ws["nkmers1_fwd"], ws["nkmers2"])
        assert t[2] == t[3] == ws["nseeds"], (t, ws["nseeds"])
        assert t[4] == ws["nhits"], (t, ws["nhits"])
        a, b = merged.canonical_lines(), whole.canonical_lines()
        assert len(a) == len(b) and a == b, (len(a), len(b))
        a, b = merged.canonical_lines_unsorted(), whole.canonical_lines_unsorted()
        if a != b:
            i = next(i for i, (x, y) in enumerate(zip(a, b)) if x != y)
            print("ORDER_MISMATCH first=%d\n  gathered %s\n  single   %s" % (i, a[i], b[i]), flush=True)
            raise AssertionError("gathered records are not in the single-GPU .1aln order")
        assert merged.nraw == whole.nraw
        key = merged.fields[:, [1, 3, 2, 0]]
        ties = int((key[1:] == key[:-1]).all(axis=1).sum())      # records whose order only the gather's tie rule sets
        print("MULTI_OK world=%d records=%d backend=%s maxicont=%d ties=%d" % (world, len(a), backend,
                                                                             int(maxic.item()), ties))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

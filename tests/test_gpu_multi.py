"""-m gpu: the N > 1 path (k-mer-space sharding, record exchanges, gather) in real multi-process runs at 2, 3,
4 and 8 ranks.  A world runs over NCCL, one GPU per rank, where the machine has a GPU for every rank, and
over gloo with every rank on the one GPU (gloo stages the device buffers through host memory) where it has
fewer.  Rank 0 checks the gathered records against a single-GPU run of the pair, in .1aln order; every
rank, including ranks that own no contig, checks that it received only seeds of A-contigs it owns.

torchrun_ranks.run bounds every run in time and stops every rank on a timeout or an interrupt, so no
rank outlives its test."""
import os
import re

import pytest

import torchrun_ranks

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_rank_sharded_run_equals_single_gpu_run():
    _ranks(2, "default", 29611)


def test_two_rank_sharded_run_routes_seeds_whose_icont_straddles_bit_64():
    """the icont_straddles case of tests/edge_cases.py: 300 A-contig ranks, and the owner routing
    reads an icont field that straddles bit 64"""
    out = _ranks(2, "icont_straddles", 29612)
    assert int(out.split("maxicont=")[1].split()[0]) > 255


@pytest.mark.parametrize("world,port", [(3, 29613), (4, 29614), (8, 29615)])
def test_sharded_run_at_more_ranks_equals_single_gpu_run(world, port):
    """uneven prefix cuts (86/85/85 top bytes at 3 ranks) and the benchmark's 4 and 8 ranks; at 8 ranks
    the six contigs of each genome leave ranks 6 and 7 without a contig to scan or a seed to extend"""
    out = _ranks(world, "default", port)
    if world == 8:
        for r in (6, 7):
            assert "RANK_OK rank=%d contigs=0 seeds=0 records=0" % r in out


def test_eight_rank_sharded_run_with_fewer_contigs_than_ranks():
    """five ranks without a contig; two copies of one A segment in B give records that tie on the gather's
    sort key, so the gathered order also pins its tie rule"""
    out = _ranks(8, "few_contigs", 29616)
    assert out.count("contigs=0 seeds=0 records=0") == 5
    assert int(out.split(" ties=")[1].split()[0]) > 0


def _ranks(world, pair, port):
    """torchrun of tests/multi_worker.py at `world` ranks; returns its output once every check passed"""
    env = dict(os.environ, FGB_MULTI_BACKEND="nccl" if _ngpu() >= world else "gloo")
    env.pop("FGB_MULTI_PAIR", None)
    if pair != "default":
        env["FGB_MULTI_PAIR"] = pair
    rc, out = torchrun_ranks.run(os.path.join(ROOT, "tests", "multi_worker.py"), world, port, env=env)
    for what in ("OWNER_MISMATCH", "ORDER_MISMATCH"):
        assert what not in out, "\n".join(l for l in out.split("\n") if what in l or l.startswith("  "))
    errors = [l for l in out.split("\n") if "Error" in l and "ChildFailedError" not in l]
    assert rc == 0 and "MULTI_OK world=%d" % world in out, "\n".join(errors[:20]) or out[-3000:]
    # ranks share the pipe: a line of one may start after a partial line of another
    assert sorted(int(r) for r in re.findall(r"RANK_OK rank=(\d+)", out)) == list(range(world)), out[-3000:]
    return out

"""-m gpu: the N > 1 path (k-mer-space sharding, record exchanges, gather) with two ranks: one per GPU
over NCCL where there are two GPUs, both on the one GPU over gloo (which stages the device buffers
through host memory) where there is one."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_two_rank_sharded_run_equals_single_gpu_run():
    _two_ranks("default", 29611)


def test_two_rank_sharded_run_routes_seeds_whose_icont_straddles_bit_64():
    """the icont_straddles case of tests/edge_cases.py: 300 A-contig ranks, and the owner routing
    reads an icont field that straddles bit 64"""
    _two_ranks("icont_straddles", 29612)


def _two_ranks(pair, port):
    env = dict(os.environ, FGB_MULTI_BACKEND="nccl" if _ngpu() >= 2 else "gloo")
    env.pop("FGB_MULTI_PAIR", None)
    if pair != "default":
        env["FGB_MULTI_PAIR"] = pair
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tests", "multi_worker.py")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    assert "OWNER_MISMATCH" not in r.stdout, [l for l in r.stdout.split("\n") if "OWNER_MISMATCH" in l]
    errors = [l for l in r.stdout.split("\n") if "Error" in l and "ChildFailedError" not in l]
    assert r.returncode == 0 and "MULTI_OK world=2" in r.stdout, "\n".join(errors[:20]) or r.stdout[-3000:]
    if pair == "icont_straddles":
        assert int(r.stdout.split("maxicont=")[1].split()[0]) > 255

#!/usr/bin/env python
"""kmer_scan_bench.py -- the sharded path's scan (lib.kmers_scan, every contig selected) on genome A of the
bench pair, both strands and forward only, two builds of the library compared in one session.

Each round runs one process per build (FGB_LIB selects it; a parent build comes from a build of the parent
commit), alternating the builds.  A process stages the genome, runs --warmup scans of each kind, then --reps
timed scans of each kind, alternating the kinds.  Per scan it takes scan_ms, the library's CUDA-event time
of the count and emit passes (stage_ms.scan_ms of bench.py), and call_ms, the host clock around the whole
call (tile list, allocations and the host wait included; the call ends in a device synchronise).  The
records of one scan of each kind are summed and XORed word by word on the host: the two builds must give
the same records, in whatever order.  Prints one JSON line; the card's name and power limit are read in the
same run.

  python profiles/kmer_scan_bench.py --lib-a fastga_b200/libfastga_b200_parent.so --lib-b fastga_b200/libfastga_b200.so \\
         --rounds 3 --reps 10 --warmup 2 --out /tmp/kmer_scan_bench_runs.json
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
KINDS = ("both", "forward")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, check=True).stdout.strip().split("\n")[0]
        name, power, mhz = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": mhz}
    except Exception as ex:
        return {"error": str(ex)[:200]}


class _DeviceRecords:
    """n 16-byte device records as a CUDA array, for torch to read"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n, 2), "typestr": "<i8", "data": (ptr, False),
                                          "strides": None, "version": 3}


def child(args):
    """one build: timed scans of genome A, one JSON line on stdout"""
    import torch
    from fastga_b200 import formats, lib
    with np.load(args.genome) as z:
        genome = formats.genome_from_arrays([z["c%d" % i] for i in range(len(z.files))])
    dg = lib.DeviceGenome(genome)
    mask = np.ones(genome.ncontig, dtype=np.uint8)

    def scan(kind, keep=False):
        lib.timings_reset()
        t0 = time.perf_counter()
        ptr, n = lib.kmers_scan(dg, mask, kind == "forward")
        call_ms = (time.perf_counter() - t0) * 1000.0
        scan_ms = lib.timings_get()["scan_ms"]
        digest = None
        if keep:
            recs = torch.as_tensor(_DeviceRecords(ptr, n), device="cuda").cpu().numpy().view(np.uint64)
            digest = [str(int(np.bitwise_xor.reduce(recs[:, k]))) + "/" + str(int(recs[:, k].sum(dtype=np.uint64)))
                      for k in (0, 1)]
        lib.device_free(ptr)
        return n, scan_ms, call_ms, digest

    out = {k: {"scan_ms": [], "call_ms": []} for k in KINDS}
    for k in KINDS:
        out[k]["n"], _, _, out[k]["digest"] = scan(k, keep=True)
    for _ in range(args.warmup):
        for k in KINDS:
            scan(k)
    for _ in range(args.reps):
        for k in KINDS:
            _, s, c, _ = scan(k)
            out[k]["scan_ms"].append(s)
            out[k]["call_ms"].append(c)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", help="the parent build")
    ap.add_argument("--lib-b", help="this build")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the runs here (JSON)")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--genome", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)

    import bench
    A, _ = bench.workload(1)
    runs = []
    with tempfile.TemporaryDirectory() as tmp:
        gpath = os.path.join(tmp, "genome_a.npz")
        np.savez(gpath, **{"c%d" % i: c for i, c in enumerate(A)})
        for r in range(args.rounds):
            rnd = {}
            for tag, lib in (("a", args.lib_a), ("b", args.lib_b)):
                env = dict(os.environ, FGB_LIB=os.path.abspath(lib))
                cmd = [sys.executable, os.path.abspath(__file__), "--child", tag, "--genome", gpath,
                       "--reps", str(args.reps), "--warmup", str(args.warmup)]
                out = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, text=True, check=True, cwd=ROOT).stdout
                rnd[tag] = json.loads(out.strip().splitlines()[-1])
            runs.append(rnd)
            print(json.dumps({"round": r, **rnd}), file=sys.stderr)

    same = all(rnd["a"][k]["n"] == rnd["b"][k]["n"] and rnd["a"][k]["digest"] == rnd["b"][k]["digest"]
               for rnd in runs for k in KINDS)
    summary = {}
    for k in KINDS:
        for m in ("scan_ms", "call_ms"):
            a = np.array([v for rnd in runs for v in rnd["a"][k][m]])
            b = np.array([v for rnd in runs for v in rnd["b"][k][m]])
            ra = [float(np.median(rnd["a"][k][m])) for rnd in runs]
            rb = [float(np.median(rnd["b"][k][m])) for rnd in runs]
            summary["%s_%s" % (k, m)] = {"a_median": float(np.median(a)), "b_median": float(np.median(b)),
                                         "a_min_max": [float(a.min()), float(a.max())],
                                         "b_min_max": [float(b.min()), float(b.max())],
                                         "a_round_medians": ra, "b_round_medians": rb}
    line = {"what": "lib.kmers_scan of bench genome A (bench.py workload, N = 1), every contig, build a vs b "
                    "alternating", "gpu": gpu_info(), "lib_a": os.path.basename(args.lib_a),
            "lib_b": os.path.basename(args.lib_b), "rounds": args.rounds, "reps": args.reps, "warmup": args.warmup,
            "records": {k: runs[0]["b"][k]["n"] for k in KINDS}, "records_same": same, "summary": summary}
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"summary": line, "runs": runs}, f, indent=1)
    print(json.dumps(line))


if __name__ == "__main__":
    main()

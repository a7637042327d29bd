#!/usr/bin/env python
"""kmer_build_bench.py -- the bench pair's two k-mer tables built from one syncmer scan along the two routes
into the k-mer sort, alternating them: "scatter", the default, where the sort starts from the scan's
layout (the records in runs by the first digit of the k-mer partition), against "partition"
(FGB_KSORT_PARTITION=1), where the sort ignores that layout and runs every partition pass in Onesweep.

The tables are the ones the fused path builds: genome A forward-only, genome B both strands.  Times are
the library's CUDA-event times (stage_ms.scan_ms + stage_ms.ksort_ms of bench.py), summed over the two
tables.  A separate profiled build of each path splits the time by kernel (torch.profiler, CUDA activity).
HBM bytes per record, counting 32-byte sectors (reading the staged genome is < 1 byte per record):
  scatter:    16 (emit in runs) + 32 (one partition pass) + 16 (bin bounds) + 32 (bucket sort) = 96
  partition:  16 (emit in runs) + 16 (histogram) + 2 x 32 (partition passes) + 16 (bin bounds) + 32 = 144
Prints one JSON line.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0          # H100 SXM data sheet, HBM3
BYTES = {"scatter": 96, "partition": 144}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, check=True).stdout.strip().split("\n")[0]
        name, power, mhz = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": mhz}
    except Exception as ex:
        return {"error": str(ex)[:200]}


def set_path(path):
    if path == "partition":
        os.environ["FGB_KSORT_PARTITION"] = "1"
    else:
        os.environ.pop("FGB_KSORT_PARTITION", None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch
    import bench
    from fastga_b200 import formats, lib

    A, B = bench.workload(1)
    gA, gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
    dA, dB = lib.DeviceGenome(gA), lib.DeviceGenome(gB)

    def build(path):
        set_path(path)
        lib.timings_reset()
        xA, xB = lib.DeviceGix.build_forward(dA), lib.DeviceGix.build(dB)
        t = lib.timings_get()
        return (xA, xB), t["scan_ms"], t["ksort_ms"]

    paths = ("scatter", "partition")
    ms = {p: {"scan": [], "ksort": []} for p in paths}
    for i in range(args.warmup + args.reps):
        for p in paths:
            xs, scan, ksort = build(p)
            for x in xs:
                x.close()
            if i >= args.warmup:
                ms[p]["scan"].append(scan)
                ms[p]["ksort"].append(ksort)

    digests, n = {}, None
    for p in paths:
        xs, _, _ = build(p)
        digests[p] = [hashlib.md5(a.tobytes()).hexdigest() for x in xs for a in x.download()]
        n = [x.n for x in xs]
        for x in xs:
            x.close()
    identical = digests["scatter"] == digests["partition"]

    kernels = {}
    for p in paths:
        for x in build(p)[0]:                           # warm
            x.close()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            xs, _, _ = build(p)
            torch.cuda.synchronize()
        for x in xs:
            x.close()
        k = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            if t > 0:
                k[e.key.split("(")[0][:60]] = round(t / 1000.0, 4)
        kernels[p] = dict(sorted(k.items(), key=lambda kv: -kv[1]))
    set_path("scatter")
    torch.cuda.synchronize()

    nrec = sum(n)

    def summary(p):
        scan, ksort = np.array(ms[p]["scan"]), np.array(ms[p]["ksort"])
        tot = scan + ksort
        med = float(np.median(tot))
        gbs = nrec * BYTES[p] / med / 1e6
        return {"scan_plus_ksort_ms_median": med, "min_max": [float(tot.min()), float(tot.max())],
                "scan_ms_median": float(np.median(scan)), "ksort_ms_median": float(np.median(ksort)),
                "reps": len(tot), "bytes_per_record": BYTES[p], "bytes": nrec * BYTES[p], "GB_s": gbs,
                "frac_of_3350_GB_s": gbs / PEAK_GBS, "kernel_ms_profiled_build": kernels[p]}

    line = {"what": "k-mer tables of the bench pair (bench.py workload, N = 1): A forward-only + B both strands",
            "gpu": gpu_info(), "records": n, "scatter": summary("scatter"), "partition": summary("partition"),
            "tables_pstart_buck_byte_identical": identical}
    line["speedup"] = line["partition"]["scan_plus_ksort_ms_median"] / line["scatter"]["scan_plus_ksort_ms_median"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""seed_sort_bench.py -- the seed sort of the bench pair on 64-bit words against the 128-bit passes.

Builds the bench pair's tables once, takes the unsorted seeds from the merge and sorts copies of them
through fgb_seeds_from_records, alternating the two paths (FGB_SEED_SORT_WIDE=1 forces the 128-bit
passes).  Times are the library's CUDA-event time of the sort alone (stage_ms.ssort_ms of bench.py).
Bytes per seed (DRAM moves 32-byte sectors, so the histogram pre-pass streams all 16 bytes):
  128-bit: 16 + 32 x passes            64-bit: 16 + (16 + 8) + 16 x (passes - 2) + (8 + 16)
Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0          # H100 SXM data sheet, HBM3


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, check=True).stdout.strip().split("\n")[0]
        name, power, mhz = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": mhz}
    except Exception as ex:
        return {"error": str(ex)[:200]}


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
    xA, xB = lib.DeviceGix.build_forward(dA), lib.DeviceGix.build(dB)
    amx, bmx = int(gA.clen.max()), int(gB.clen.max())
    ptr, n, bits, sumlen, _ = lib.seeds_merge(xA, xB, amx, bmx, 10)
    xA.close()
    xB.close()
    key = 12 + sum(bits) + 1
    passes = (key - 6 + 7) // 8

    def run(wide):
        if wide:
            os.environ["FGB_SEED_SORT_WIDE"] = "1"
        else:
            os.environ.pop("FGB_SEED_SORT_WIDE", None)
        lib.timings_reset()
        s = lib.seeds_from_records(ptr, n, bits, amx, bmx, sumlen)
        ms = lib.timings_get()["ssort_ms"]
        return s, ms

    ms = {False: [], True: []}
    for i in range(args.warmup + args.reps):
        for wide in (False, True):
            s, t = run(wide)
            s.close()
            if i >= args.warmup:
                ms[wide].append(t)
    s64, _ = run(False)
    s128, _ = run(True)
    os.environ.pop("FGB_SEED_SORT_WIDE", None)
    identical = s64.download().tobytes() == s128.download().tobytes()
    s64.close()
    s128.close()
    lib.device_free(ptr)
    torch.cuda.synchronize()

    def summary(wide):
        v = np.array(ms[wide])
        per = 16 + 32 * passes if wide else 16 + 24 + 16 * (passes - 2) + 24
        med = float(np.median(v))
        gbs = n * per / med / 1e6
        return {"ms_median": med, "ms_min_max": [float(v.min()), float(v.max())], "reps": len(v),
                "bytes_per_seed": per, "bytes": n * per, "GB_s": gbs, "frac_of_3350_GB_s": gbs / PEAK_GBS}

    line = {"what": "seed sort of the bench pair (bench.py workload, N = 1), fgb_seeds_from_records",
            "gpu": gpu_info(), "seeds": n, "key_bits": key, "passes": passes,
            "sort64": summary(False), "sort128": summary(True), "outputs_byte_identical": identical}
    line["speedup"] = line["sort128"]["ms_median"] / line["sort64"]["ms_median"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()

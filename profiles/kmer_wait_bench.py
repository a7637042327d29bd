#!/usr/bin/env python
"""kmer_wait_bench.py -- the two k-mer table builds of the bench pair (syncmer scan to merge launch), two
builds of the library compared in one session.

Runs `bench.py --gpus 1` alternately with each library (FGB_LIB; a parent build comes from
profiles/build_variant.sh or a build of the parent commit), --pairs times.  The first pair also runs the
reference (parity) and dumps both builds' alignments, which must be byte-identical.  Per run it takes:
  us_gix    host_wall_us us_gix in ms: the host clock from the first scan to the merge launch, every host
            wait and host loop of the two table builds included
  scan_ms, ksort_ms, index_ms   stage_ms: CUDA-event time of the scan, the k-mer sort and the prefix index
  step_ms   bench.py's step median
Prints one JSON line; the card's name and power limit are read in the same run.

  python profiles/kmer_wait_bench.py --lib-a fastga_b200/libfastga_b200_parent.so --lib-b fastga_b200/libfastga_b200.so \
         --pairs 6 --steps 10 --warmup 3 --out /tmp/kmer_wait_bench_runs.json
"""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, check=True).stdout.strip().split("\n")[0]
        name, power, mhz = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": mhz}
    except Exception as ex:
        return {"error": str(ex)[:200]}


def run_bench(lib, steps, warmup, reference, dump):
    env = dict(os.environ, FGB_LIB=os.path.abspath(lib))
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps),
           "--warmup", str(warmup)]
    if not reference:
        cmd.append("--no-cpu-baseline")
    if dump:
        cmd += ["--dump-outputs", dump]
    out = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, text=True, check=True, cwd=ROOT).stdout
    line = json.loads([s for s in out.splitlines() if s.startswith("{")][-1])
    c = line["config"]
    st, hw = c["stage_ms"], c["host_wall_us"]
    return {"step_ms": c["step_ms_min_med_max"][1], "step_ms_min_med_max": c["step_ms_min_med_max"],
            "us_gix": hw["us_gix"] / 1000.0, "scan_ms": st["scan_ms"], "ksort_ms": st["ksort_ms"],
            "index_ms": st["index_ms"], "kmers": c["kmers"], "seeds": c["seeds"], "hits": c["hits"], "triples": c["triples"],
            "waves": c["waves"], "aln_md5": c["aln_md5"], "gpu_launches": line["gpu_launches"],
            "parity_equal": line.get("parity", {}).get("equal")}


def dumps_identical(da, db):
    fa, fb = sorted(os.listdir(da)), sorted(os.listdir(db))
    return fa == fb and len(fa) > 0 and all(filecmp.cmp(os.path.join(da, f), os.path.join(db, f), shallow=False)
                                            for f in fa)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", required=True, help="the parent build")
    ap.add_argument("--lib-b", required=True, help="this build")
    ap.add_argument("--pairs", type=int, default=6)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the runs here (JSON)")
    args = ap.parse_args()

    runs = []
    with tempfile.TemporaryDirectory() as tmp:
        for p in range(args.pairs):
            pair = {}
            for tag, lib in (("a", args.lib_a), ("b", args.lib_b)):
                dump = os.path.join(tmp, tag) if p == 0 else None
                pair[tag] = run_bench(lib, args.steps, args.warmup, p == 0, dump)
            if p == 0:
                pair["dumps_identical"] = dumps_identical(os.path.join(tmp, "a"), os.path.join(tmp, "b"))
            runs.append(pair)
            print(json.dumps({"pair": p, **pair}), file=sys.stderr)

    def col(tag, k):
        return np.array([r[tag][k] for r in runs], dtype=float)

    same = all(r["a"][k] == r["b"][k] for r in runs for k in ("kmers", "seeds", "hits", "triples", "waves", "aln_md5"))
    summary = {}
    for k in ("us_gix", "scan_ms", "ksort_ms", "index_ms", "step_ms"):
        a, b = col("a", k), col("b", k)
        summary[k] = {"a_median": float(np.median(a)), "b_median": float(np.median(b)),
                      "a_min_max": [float(a.min()), float(a.max())], "b_min_max": [float(b.min()), float(b.max())],
                      "b_lower_in_every_pair": bool((b < a).all()), "pair_diff_min_max": [float((a - b).min()),
                                                                                          float((a - b).max())]}
    line = {"what": "k-mer table builds of the bench pair (bench.py --gpus 1), build a vs b alternating",
            "gpu": gpu_info(), "lib_a": os.path.basename(args.lib_a), "lib_b": os.path.basename(args.lib_b),
            "pairs": args.pairs, "steps": args.steps, "warmup": args.warmup,
            "outputs_same": same, "dumps_identical": runs[0].get("dumps_identical"),
            "parity_equal": [runs[0]["a"]["parity_equal"], runs[0]["b"]["parity_equal"]],
            "summary": summary}
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"summary": line, "runs": runs}, f, indent=1)
    print(json.dumps(line))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Time the reference's single-GPU C+CUDA PFSP driver as it builds it (oracle/_ref/pfsp_gpu_cuda.out, its own
evaluate.cu for sm_90a) against the same driver relinked against libtsb200_cbase.so (pfsp_gpu_cuda_tsb.out), both
from oracle/cbase.mk.  The two binaries run alternately, `--reps` times each per case, and the tool reports the
drivers' own timers: the step-2 "Elapsed time" (the GPU loop, where the evaluate_gpu calls are) and the total of the
final report, with the counts, which must be equal.  One JSON line per case, preceded by the card's name, power limit
and max SM clock, which belong beside every time.

    python tools/cbase_time.py [--reps 3] [--cases ta014:lb1,ta011:lb1_d,ta014:lb2] [--m 25] [--M 50000]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_OUT = os.path.join(ROOT, "oracle", "_ref")
LBS = {"lb1_d": 0, "lb1": 1, "lb2": 2}


def run(exe, inst, lb, m, M):
    with tempfile.TemporaryDirectory() as cwd:  # (the driver appends to a stats file in its working directory)
        r = subprocess.run([exe, "--inst", str(inst), "--lb", str(LBS[lb]), "--ub", "1", "--m", str(m), "--M", str(M)],
                           capture_output=True, text=True, cwd=cwd, check=True)
    if "tsb200_cbase" in r.stderr:
        raise RuntimeError(r.stderr)
    out = r.stdout
    step2 = float(re.search(r"Search on GPU completed\n.*?Elapsed time: ([\d.]+)", out, re.S).group(1))
    last = lambda pat: re.findall(pat, out)[-1]  # noqa: E731
    return {"step2_s": step2, "total_s": float(last(r"Elapsed time: ([\d.]+) \[s\]")),
            "counts": [int(last(r"explored tree: (\d+)")), int(last(r"explored solutions: (\d+)")),
                       int(last(r"makespan: (\d+)"))]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cases", default="ta014:lb1,ta011:lb1_d,ta014:lb2")
    ap.add_argument("--m", type=int, default=25)
    ap.add_argument("--M", type=int, default=50000)
    a = ap.parse_args()
    exes = {"original": os.path.join(REF_OUT, "pfsp_gpu_cuda.out"), "relinked": os.path.join(REF_OUT, "pfsp_gpu_cuda_tsb.out")}
    for e in exes.values():
        if not os.path.exists(e):
            sys.exit(f"{e} is missing: build() makes it where a checkout of the reference exists")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card, "m": a.m, "M": a.M, "reps": a.reps}), flush=True)
    for case in a.cases.split(","):
        tag, lb = case.split(":")
        inst = int(tag[2:])
        res = {k: [] for k in exes}
        run(exes["original"], inst, lb, a.m, a.M)  # warm-up: module loading, the first context of the process
        for _ in range(a.reps):
            for k, e in exes.items():
                res[k].append(run(e, inst, lb, a.m, a.M))
        counts = {tuple(r["counts"]) for rs in res.values() for r in rs}
        print(json.dumps({"case": case, "same_counts": len(counts) == 1, "counts": list(counts.pop()),
                          **{f"{k}_step2_s": [r["step2_s"] for r in rs] for k, rs in res.items()},
                          **{f"{k}_total_s": [r["total_s"] for r in rs] for k, rs in res.items()}}), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Counts of whole PFSP searches as the reference's sequential C program prints them (oracle/_ref/pfsp_c.out: the C
baseline's min_heads, which its C+CUDA drivers share), under --ub 1, for the instances and bounds that finish in
seconds on one CPU core.  Under ub = 1 the incumbent never falls, so a node is explored iff its bound is below the
optimum whatever the order: the explored tree, explored solutions and optimum are the same for the GPU drivers at any
--m, --M, --D and --perc.  tests/test_gpu_cbase.py checks the relinked drivers (oracle/cbase.mk) against them.

Needs a checkout of the reference (oracle/Makefile: $TSB200_REFERENCE, by default `reference` next to this
repository):  make -C oracle _ref/pfsp_c.out && python tests/golden/make_golden_cbase.py
"""
import json
import os
import re
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pfsp_cbase_searches.json")
EXE = os.path.join(ROOT, "oracle", "_ref", "pfsp_c.out")
# ta001, 005, 006, 008, 010, 017, 020 and 021 take longer than 15 s each with lb1 on one core: left out
INSTANCES = (2, 3, 4, 7, 9, 11, 14)
LBS = {"lb1_d": 0, "lb1": 1, "lb2": 2}


def parse(txt):
    """the counts of the final report of the reference's PFSP programs (print_results)"""
    g = lambda pat: int(re.findall(pat, txt)[-1])  # noqa: E731
    return {"tree": g(r"Size of the explored tree: (\d+)"), "sol": g(r"Number of explored solutions: (\d+)"),
            "best": g(r"Optimal makespan: (\d+)")}


def run(inst, lb, exe=EXE):
    # (the reference's programs append to a stats file in their working directory)
    with tempfile.TemporaryDirectory() as cwd:
        txt = subprocess.run([exe, "--inst", str(inst), "--lb", str(lb), "--ub", "1"], capture_output=True, text=True,
                             cwd=cwd, check=True).stdout
    return parse(txt)


def main():
    jobs = [(inst, name) for inst in INSTANCES for name in LBS]
    with ThreadPoolExecutor(max_workers=os.cpu_count()) as ex:
        res = list(ex.map(lambda j: run(j[0], LBS[j[1]]), jobs))
    out = {"_source": "oracle/_ref/pfsp_c.out (the reference's sequential C program) --ub 1",
           "searches": {f"ta{inst:03d}_{name}": r for (inst, name), r in zip(jobs, res)}}
    json.dump(out, open(OUT, "w"), indent=1)
    print("wrote", OUT, file=sys.stderr)


if __name__ == "__main__":
    main()

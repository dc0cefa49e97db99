#!/usr/bin/env python
"""Counts of whole 50-job PFSP searches (ta031..ta060) as the reference's sequential C program built with
MAX_JOBS = 50 prints them, under --ub 1, for the instances whose search finishes at once: ta032, ta037 and ta038 with
lb1, lb1_d and lb2 (every other 50-job instance runs for minutes or more with every bound).

The program is the reference's pfsp_c.c compiled from the oracle's MAX_JOBS = 50 copy of its PFSP sources
(oracle/Makefile, _ref/jobs50) with the Chapel program's min_heads (_ref/chapel_sem/c_bound_simple.c, SURVEY.md
Appendix A.1): the library follows the Chapel program, and with the C baseline's min_heads lb1_d explores 11 and 1
nodes on ta037 and ta038 where the Chapel rule explores none.  Under ub = 1 the incumbent never falls, so the counts
are the same for every --m, --M, --D and number of pools.  tests/test_gpu_pfsp50_search.py checks the 50-job searches
against them.

Needs a checkout of the reference:  make -C oracle ref && python tests/golden/make_golden_pfsp50.py
"""
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_cbase import parse  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pfsp50_searches.json")
REF = os.path.join(ROOT, "oracle", "_ref")
INSTANCES = (32, 37, 38)
LBS = {"lb1_d": 0, "lb1": 1, "lb2": 2}


def build(exe):
    j50 = os.path.join(REF, "jobs50")
    lib = os.path.join(j50, "pfsp", "lib")
    srcs = [os.path.join(j50, "pfsp", "pfsp_c.c")] + [os.path.join(lib, f) for f in (
        "c_taillard.c", "c_bound_johnson.c", "PFSP_node.c", "Pool.c")] + [
        os.path.join(REF, "chapel_sem", "c_bound_simple.c"), os.path.join(j50, "commons", "util.c")]
    # (-I: the MAX_JOBS = 50 headers for the Chapel-semantics c_bound_simple.c too)
    subprocess.run(["gcc", "-O3", "-w", f"-I{lib}", "-o", exe, *srcs, "-lm"], check=True)


def main():
    out = {"_source": "the reference's pfsp_c.c with MAX_JOBS = 50 and the Chapel program's min_heads "
                      "(oracle/_ref/jobs50 + oracle/_ref/chapel_sem) --ub 1", "searches": {}}
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "pfsp_c50.out")
        build(exe)
        for inst in INSTANCES:
            for name, lb in LBS.items():
                # (the reference's programs append to a stats file in their working directory)
                txt = subprocess.run([exe, "--inst", str(inst), "--lb", str(lb), "--ub", "1"], capture_output=True,
                                     text=True, cwd=tmp, check=True, timeout=600).stdout
                out["searches"][f"ta{inst:03d}_{name}"] = parse(txt)
    json.dump(out, open(OUT, "w"), indent=1)
    print("wrote", OUT, file=sys.stderr)


if __name__ == "__main__":
    main()

"""What the resumable searches (tsb_*_search_device_ckpt on device pools, tsb_*_search_ckpt on host pools) cost when
they do not stop, what a stop costs, and how large their checkpoints are.

  python tools/search_ckpt_time.py [--reps 3] [--parts whole,capped,checkpoints,host] [--out DIR]

1. Whole searches, the twin and the resumable search without a time limit alternated `reps` times on warm handles
   (step-2 seconds and kernel launches): N = 17 at M = 50 000 (four pools per task, 2048 rounds per call in both) and
   ta014 lb1 at M = 50 000 (one pool: the resumable search caps its calls at 1024 rounds).
2. The capped calls on the larger golden N = 21 subtree (tests/golden/nqueens_wide.json) at M = 50 000 on a warm wide
   handle: one unbounded pool_run against loops of 1024 rounds (the cap) and of 16 rounds (to show the cost of a
   call boundary), alternated `reps` times.
3. Checkpoints: N = 17, the whole N = 21 search and ta014 lb1, all at M = 50 000, stopped after `--stop` seconds
   (N = 17, ta014: after one call), with the file's size, the time from the stop to the return, the write and read
   times (TSB200_TRACE lines of a child process) and the time of the resumed invocation.
4. Host pools: the twin (tsb_pfsp_search, tsb_nq_search) and its resumable form without a time limit alternated `reps`
   times, ta014 lb1 and N = 17 (--host-N; about three minutes per search on an H100), both at M = 50 000 (step-2
   seconds): the resumable form asks for a stop once per chunk.
Prints one JSON line per measurement after the name and power limit of the card; --out DIR also writes them to
DIR/search_ckpt_time.jsonl."""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tsb200  # noqa: E402
from tsb200 import _lib  # noqa: E402

LINES = []


def emit(d):
    LINES.append(d)
    print(json.dumps(d), flush=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "(nvidia-smi gave no answer)"


def nq_ckpt(path, N, M, seconds, max_queens=20):
    st = _lib.SearchStats()
    rc = tsb200.lib().tsb_nq_search_device_ckpt(max_queens, N, 1, 25, M, 1, os.fsencode(path), seconds, C.byref(st))
    return rc, st


def pfsp_ckpt(path, M, seconds):
    st = _lib.SearchStats()
    rc = tsb200.lib().tsb_pfsp_search_device_ckpt(14, 1, 1, 25, M, 1, 1, os.fsencode(path), seconds, C.byref(st))
    return rc, st


def whole(reps, tmp):
    cases = {
        "nq17_M50000": (lambda: tsb200.nqueens_search_device(17, 1, 25, 50000, 1),
                        lambda p: nq_ckpt(p, 17, 50000, -1.0)),
        "ta014_lb1_M50000": (lambda: tsb200.pfsp_search_device(14, "lb1", 1, 25, 50000, 1),
                             lambda p: pfsp_ckpt(p, 50000, -1.0)),
    }
    for name, (twin, ckpt) in cases.items():
        twin()
        ckpt(os.path.join(tmp, "warm"))
        for rep in range(reps):
            a = twin()
            rc, b = ckpt(os.path.join(tmp, name))
            assert rc == _lib.OK and (a.explored_tree, a.explored_sol, a.best) == (b.explored_tree, b.explored_sol, b.best)
            emit({"what": "whole search", "case": name, "rep": rep, "twin_step2_s": round(a.t_step2, 5),
                  "ckpt_step2_s": round(b.t_step2, 5), "twin_launches": a.kernel_launches,
                  "ckpt_launches": b.kernel_launches, "offloads": a.offloads})


def host_whole(reps, tmp, N):
    cases = {
        "host_ta014_lb1_M50000": (lambda: tsb200.pfsp_search(14, "lb1", 1, 25, 50000, 1),
                                  lambda p: tsb200.pfsp_search(14, "lb1", 1, 25, 50000, 1, checkpoint=p)),
        f"host_nq{N}_M50000": (lambda: tsb200.nqueens_search(N, 1, 25, 50000, 1),
                               lambda p: tsb200.nqueens_search(N, 1, 25, 50000, 1, checkpoint=p)),
    }
    for name, (twin, ckpt) in cases.items():
        for rep in range(reps):
            a = twin()
            b = ckpt(os.path.join(tmp, name))
            assert (a.explored_tree, a.explored_sol, a.best, a.offloads) == \
                (b.explored_tree, b.explored_sol, b.best, b.offloads)
            emit({"what": "whole host-pool search", "case": name, "rep": rep, "twin_step2_s": round(a.t_step2, 4),
                  "ckpt_step2_s": round(b.t_step2, 4), "offloads": a.offloads,
                  "twin_Mnodes_per_s": round(a.explored_tree / a.t_step2 / 1e6, 2),
                  "ckpt_Mnodes_per_s": round(b.explored_tree / b.t_step2 / 1e6, 2)})


def capped(reps):
    import nq_wide_rounds as w
    sub = max((s for s in w.GOLDEN if s["N"] == 21), key=lambda s: s["tree"])
    M = 50000
    with tsb200.NQueensEvaluator(21, M=M, max_queens=24) as ev:
        def run(cap):
            ev.pool_push(w.subtree_root(21, sub["prefix"], True))
            calls, tot = 0, [0, 0, 0, 0]
            t0 = time.perf_counter()
            while True:
                r = ev.pool_run(1, M, cap)
                calls += 1
                tot = [x + int(y) for x, y in zip(tot, r)]
                if ev.pool_size < 1 or int(r[0]) < cap:
                    break
            return time.perf_counter() - t0, calls, tot
        run(2**62)
        for rep in range(reps):
            res = {cap: run(cap) for cap in (2**62, 1024, 16)}
            base = res[2**62][2]
            assert all(r[2] == base for r in res.values()), res
            emit({"what": "capped calls, N = 21 subtree", "prefix": sub["prefix"], "M": M, "rep": rep, "rounds": base[0],
                  "unbounded_s": round(res[2**62][0], 5), "cap1024_s": round(res[1024][0], 5),
                  "cap1024_calls": res[1024][1], "cap16_s": round(res[16][0], 5), "cap16_calls": res[16][1]})


CHILD = """
import ctypes as C, os, sys, time
sys.path.insert(0, {pkg!r})
import tsb200
from tsb200 import _lib
L = tsb200.lib()
kind, path, seconds = sys.argv[1], sys.argv[2].encode(), float(sys.argv[3])
st = _lib.SearchStats()
t0 = time.perf_counter()
if kind == "nq17":
    rc = L.tsb_nq_search_device_ckpt(20, 17, 1, 25, 50000, 1, path, seconds, C.byref(st))
elif kind == "nq21":
    rc = L.tsb_nq_search_device_ckpt(20, 21, 1, 25, 50000, 1, path, seconds, C.byref(st))
else:
    rc = L.tsb_pfsp_search_device_ckpt(14, 1, 1, 25, 50000, 1, 1, path, seconds, C.byref(st))
print("RESULT", rc, time.perf_counter() - t0, st.explored_tree, st.t_step1, st.t_step2)
"""


def checkpoints(tmp, stop21):
    env = dict(os.environ, TSB200_TRACE="1")
    code = CHILD.format(pkg=os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200"))
    for kind, seconds in (("nq17", 0.0), ("ta014", 0.0), ("nq21", stop21)):
        path = os.path.join(tmp, kind + ".ck")
        runs = []
        for leg, s in (("stop", seconds), ("resume", seconds)):
            p = subprocess.run([sys.executable, "-c", code, kind, path, str(s)], env=env, capture_output=True, text=True)
            m = re.search(r"RESULT (-?\d+) (\S+) (\d+) (\S+) (\S+)", p.stdout)
            if not m:
                raise SystemExit(p.stdout + p.stderr)
            wrote = re.findall(r"checkpoint: (\d+) nodes written in (\S+) ms", p.stderr)
            read = re.findall(r"checkpoint: read in (\S+) ms", p.stderr)
            runs.append({"leg": leg, "rc": int(m.group(1)), "call_s": round(float(m.group(2)), 4),
                         "tree_so_far": int(m.group(3)), "bytes": os.path.getsize(path) if os.path.exists(path) else 0,
                         "nodes_written": int(wrote[-1][0]) if wrote else 0,
                         "write_ms": float(wrote[-1][1]) if wrote else None,
                         "read_ms": float(read[-1]) if read else None})
        emit({"what": "checkpoint", "case": kind, "seconds": seconds, "legs": runs})
        if os.path.exists(path):
            os.remove(path)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--stop", type=float, default=5.0, help="seconds of the N = 21 search before it stops")
    ap.add_argument("--host-N", type=int, default=17, help="board size of the host-pool N-Queens case")
    ap.add_argument("--parts", default="whole,capped,checkpoints,host", help="which measurements, comma-separated")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    parts = a.parts.split(",")
    emit({"card": card()})
    with tempfile.TemporaryDirectory() as tmp:
        if "whole" in parts:
            whole(a.reps, tmp)
        if "capped" in parts:
            capped(a.reps)
        if "checkpoints" in parts:
            checkpoints(tmp, a.stop)
        if "host" in parts:
            host_whole(a.reps, tmp, a.host_N)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "search_ckpt_time.jsonl"), "w") as f:
            f.writelines(json.dumps(d) + "\n" for d in LINES)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""What paces the shared launches of bench.py's headline step 2 (N-Queens N=17 m=25 --M 50000, four device pools).

python tools/step2_pace.py [--steps 3] [--launches]

Replays bench.py's step2() on one GPU: the same warm-up split into P pools (the reference's strided split), the same
calls of tsb_nq_pool_run_multi with 2048 rounds per pool, the same steal rule between calls (a pool with fewer than m
nodes takes the oldest half of the fullest pool).  It runs with TSB200_ROUNDS_PROF=1 and reads the library's per-launch
records from stderr (NqRounds::report: "LL pace", "LL residency").  A launch ends when its last pool leaves; the other
pools idle their CTAs' share of the GPU for the rest of it.  After one step that warms up, per timed step:
  launches, steals, the time inside launches (first pool start to last pool exit, %globaltimer) against t_dev (CUDA
  events around the whole step), and the host time between launches (last exit of one launch to the first start of
  the next: synchronisation, the host's bookkeeping and the profile's own printing, and the launch)
Per pool over the timed steps: rounds, period (wall time from its start to its exit over its rounds), idle share of the
launches' time, launches it left last, why it left (budget: its 2048-round budget; dry: fewer than m nodes; relaunch:
layer table or tag window; space: arena room), and CTA 0's cycles per round in each phase.
--launches: one line per launch as well (which pool left last, each pool's exit and idle share)."""
import argparse
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200")]

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--launches", action="store_true")
ap.add_argument("--mhz", type=float, default=1980.0, help="SM clock that converts the periods to cycles")
ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
a = ap.parse_args()


def child():
    """bench.py's step 2, with markers on stderr between the library's records"""
    import numpy as np
    import torch

    import tsb200
    from bench import M_HEAD, N_HEAD, m_HEAD

    def mark(s):
        sys.stderr.flush()
        print(f"[step2_pace] {s}", file=sys.stderr, flush=True)

    N, M, m = N_HEAD, M_HEAD, m_HEAD
    torch.cuda.set_device(0)
    ev = tsb200.NQueensEvaluator(N, 1, M, device=0)
    P = max(1, min(int(os.environ.get("TSB200_POOLS", "4")), ev.pools_per_launch(M)))
    evs = [ev] + [tsb200.NQueensEvaluator(N, 1, M, device=0) for _ in range(P - 1)]
    warm, _, _ = tsb200.nqueens_warmup(N, P * m)
    c = warm.shape[0] // P
    parts = [np.ascontiguousarray(warm[g:P * c:P]) for g in range(P)]
    parts[-1] = np.ascontiguousarray(np.concatenate([parts[-1], warm[P * c:]]))
    floor = 2 * m
    stream = torch.cuda.ExternalStream(ev.stream, device=torch.device("cuda:0"))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for step in range(a.steps + 1):
        for e, part in zip(evs, parts):
            e.pool_push(part)
        torch.cuda.synchronize()
        mark(f"step {step} begin")
        per_pool = np.zeros((P, 4), dtype=np.int64)
        e0.record(stream)
        while True:
            sizes = [e.pool_size for e in evs]
            for i, e in enumerate(evs):
                if sizes[i] < m:
                    v = max(range(P), key=lambda j: sizes[j])
                    if v != i and sizes[v] >= floor:
                        e.pool_steal_from(evs[v], m)
                        mark(f"steal {i} <- {v}")
                        sizes = [x.pool_size for x in evs]
            if max(sizes) < m:
                break
            mark("call")
            for i, r in enumerate(tsb200.nqueens_pool_run_multi(evs, m, M, 2048)):
                per_pool[i] += r
        e1.record(stream)
        torch.cuda.synchronize()
        for e in evs:
            e.pool_drain()
        mark(f"step {step} end t_dev {e0.elapsed_time(e1):.3f} ms per pool (rounds, parents, children, solutions) "
             + " ".join(",".join(str(int(x)) for x in row) for row in per_pool))
    for e in evs:
        e.close()


if a.child:
    child()
    sys.exit(0)

env = dict(os.environ, TSB200_ROUNDS_PROF="1")
cmd = [sys.executable, os.path.abspath(__file__), "--child", "--steps", str(a.steps)]
out = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout

PHASE = re.compile(r"LL rounds kernel \(pool (\d+) of (\d+)\): (\d+) rounds; CTA 0 cycles per round: (.*)")
PACE = re.compile(r"LL pace \(pool (\d+) of (\d+), handle (\d+)\): start \+([\d.]+) us, wall ([\d.]+) us, (\d+) rounds, "
                  r".* exit (\w+), globaltimer (\d+)\.\.(\d+) ns")
RES = re.compile(r"LL residency: ")
MARK = re.compile(r"\[step2_pace\] (.*)")


def new_pool():
    return {"rounds": 0, "wall": 0.0, "idle": 0.0, "span": 0.0, "last": 0, "exits": collections.Counter(),
            "phases": collections.Counter(), "phase_rounds": 0}


pools = collections.defaultdict(new_pool)
steps = []  # per timed step: dict
step = None
launch, phase_of = [], {}
for line in out.splitlines():
    m = MARK.search(line)
    if m:
        s = m.group(1)
        if s.endswith("begin"):
            step = {"n": int(s.split()[1]), "launches": [], "steals": 0, "calls": 0}
        elif s.startswith("steal"):
            step["steals"] += 1
        elif s == "call":
            step["calls"] += 1
        elif " end " in s:
            step["t_dev"] = float(re.search(r"t_dev ([\d.]+) ms", s).group(1))
            step["counts"] = s.split("solutions) ", 1)[1]
            if step["n"] > 0:
                steps.append(step)
            step = None
        continue
    m = PHASE.search(line)
    if m:
        ph = {}
        for part in m.group(4).split("|"):
            who = "x:" if "exchange" in part else ""
            for name, val in re.findall(r"([a-z+\-]+) ([\d.]+)", part.split(":", 1)[1]):
                ph[who + name] = float(val)
        phase_of[int(m.group(1))] = (int(m.group(3)), ph)
        continue
    m = PACE.search(line)
    if m:
        launch.append({"slot": int(m.group(1)), "pool": int(m.group(3)), "wall": float(m.group(5)),
                       "rounds": int(m.group(6)), "exit": m.group(7), "t0": int(m.group(8)), "t1": int(m.group(9))})
        continue
    if RES.search(line):
        if step is not None and launch:
            t0 = min(x["t0"] for x in launch)
            t1 = max(x["t1"] for x in launch)
            last = max(launch, key=lambda x: x["t1"])["pool"]
            step["launches"].append({"t0": t0, "t1": t1, "last": last, "pools": launch})
            if step["n"] > 0:
                for x in launch:
                    p = pools[x["pool"]]
                    p["rounds"] += x["rounds"]
                    p["wall"] += x["wall"]
                    p["idle"] += 1e-3 * (t1 - x["t1"])
                    p["span"] += 1e-3 * (t1 - t0)
                    p["exits"][x["exit"]] += 1
                    p["last"] += x["pool"] == last
                    pr, ph = phase_of.get(x["slot"], (0, {}))
                    for k, v in ph.items():
                        p["phases"][k] += v * pr
                    p["phase_rounds"] += pr
        launch, phase_of = [], {}

if not steps:
    sys.exit("no timed step in the child's output:\n" + out[-4000:])
print(f"step 2 of N=17 m=25 --M 50000, {len(pools)} pools, 2048 rounds per pool per call; {len(steps)} timed steps "
      "after one that warms up (TSB200_ROUNDS_PROF=1)")
print(f"{'step':>4} {'calls':>5} {'launches':>8} {'steals':>6} {'t_dev ms':>9} {'in launches ms':>14} {'between ms':>10} "
      f"{'pool-rounds':>11}  per pool (rounds, parents, children, solutions)")
for s in steps:
    L = s["launches"]
    inside = sum(1e-6 * (x["t1"] - x["t0"]) for x in L)
    gaps = sum(1e-6 * (L[i + 1]["t0"] - L[i]["t1"]) for i in range(len(L) - 1))
    rounds = sum(x["rounds"] for y in L for x in y["pools"])
    print(f"{s['n']:>4} {s['calls']:>5} {len(L):>8} {s['steals']:>6} {s['t_dev']:>9.2f} {inside:>14.2f} {gaps:>10.2f} "
          f"{rounds:>11}  {s['counts']}")
    if a.launches:
        for i, x in enumerate(L):
            span = 1e-3 * (x["t1"] - x["t0"])
            gap = 1e-3 * (L[i + 1]["t0"] - x["t1"]) if i + 1 < len(L) else float("nan")
            ps = "  ".join(f"{p['pool']}:{p['rounds']}r {p['exit']} idle {1e-3 * (x['t1'] - p['t1']) / max(span, 1e-9):.1%}"
                           for p in sorted(x["pools"], key=lambda p: p["pool"]))
            print(f"      launch {i:>2}: {span:>9.1f} us, last pool {x['last']}, then {gap:>7.1f} us on the host | {ps}")
print(f"\n{'pool':>4} {'rounds':>8} {'period us':>10} {'cycles':>7} {'idle':>6} {'left last':>9}  exits")
for h in sorted(pools):
    p = pools[h]
    per = p["wall"] / max(1, p["rounds"])
    ex = ", ".join(f"{k} {v}" for k, v in sorted(p["exits"].items()))
    print(f"{h:>4} {p['rounds']:>8} {per:>10.4f} {per * a.mhz:>7.0f} {p['idle'] / max(p['span'], 1e-9):>6.1%} "
          f"{p['last']:>9}  {ex}")
names = list(dict.fromkeys(k for p in pools.values() for k in p["phases"]))
if names:
    print("\nCTA 0 cycles per round by phase (x: exchange warp)")
    print(f"{'phase':>22} " + " ".join(f"{h:>7}" for h in sorted(pools)))
    for k in names:
        print(f"{k:>22} " + " ".join(f"{pools[h]['phases'][k] / max(1, pools[h]['phase_rounds']):>7.0f}"
                                      for h in sorted(pools)))

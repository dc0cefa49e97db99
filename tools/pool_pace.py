#!/usr/bin/env python
"""The pace of the pools of a shared launch of the persistent N-Queens kernel (tsb_nq_pool_run_multi).

python tools/pool_pace.py [N M K reps] [--mhz 1980]   (default 17 50000 4 3)

Runs tools/multi_pool.py N M K reps with TSB200_ROUNDS_PROF=1 and reads the kernel's per-launch records from stderr.
A launch ends when its last pool leaves, so that pool sets the pace (its rounds x its period) and the others idle
their CTAs' share of the SMs after they leave.  Per pool (runs after the first, which warms up):
  period        wall time from the pool's start to its exit over its rounds (CTA 0's exchange warp, %globaltimer)
  idle          share of the launches' time the pool spent after leaving, waiting for the last pool
  children per parent / per round   from the pool's own counters: does a slow pool do more work per round, or the
                same work issued more slowly
  fertile parents   share of the pool's parents that had at least one child (all CTAs)
  wide CTA rounds   rounds of a CTA whose children took more than one staging window (LL_CAP), summed over CTAs
  phases        the cycles per round in each phase of the pool's CTA 0 (of its half of CTA 0 with four pools, which
                share a CTA two by two: nq_rounds_ll_kernel's HALVES), averaged over the pool's rounds
and which pools share an SM (%smid): two CTAs of different pools with two or three pools per launch, with the pool
whose CTA started first there; the two halves of one CTA with four."""
import argparse
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ap = argparse.ArgumentParser()
ap.add_argument("args", nargs="*", type=int, help="N M K reps")
ap.add_argument("--mhz", type=float, default=1980.0, help="SM clock that converts the periods to cycles")
a = ap.parse_args()
N, M, K, reps = (a.args + [17, 50000, 4, 3][len(a.args):])[:4]

env = dict(os.environ, TSB200_ROUNDS_PROF="1")
cmd = [sys.executable, os.path.join(ROOT, "tools", "multi_pool.py"), str(N), str(M), str(K), str(reps)]
out = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout

PHASE = re.compile(r"LL rounds kernel \(pool (\d+) of (\d+)\): (\d+) rounds; CTA 0 cycles per round: (.*)")
PACE = re.compile(r"LL pace \(pool (\d+) of (\d+), handle (\d+)\): start \+([\d.]+) us, wall ([\d.]+) us, (\d+) rounds, "
                  r"[\d.]+ us per round, stagger ([\d.]+) us, parents (\d+), children (\d+)")
EXTRA = re.compile(r"parents with children (\d+), CTA rounds over one window (\d+)")
RES = re.compile(r"LL residency: (.*)")
RUN = re.compile(r"N=\d+ M=\d+ K=\d+: .*\s([\d.]+) ms\s")


def new_pool():
    return {"rounds": 0, "wall": 0.0, "idle": 0.0, "span": 0.0, "parents": 0, "children": 0, "fertile": 0,
            "wide": 0, "phases": collections.Counter()}


pools = collections.defaultdict(new_pool)
residency = collections.Counter()
runs_ms = []
run = 0
phase_of = {}  # pool slot of the current launch -> (rounds, {phase: cycles per round})
launch = []
for line in out.splitlines():
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
        launch.append((m, EXTRA.search(line)))
        continue
    m = RES.search(line)
    if m:
        if launch and run > 0:
            span = max(float(x.group(5)) + float(x.group(4)) + float(x.group(7)) for x, _ in launch)
            for x, ex in launch:
                p = pools[int(x.group(3))]
                r = int(x.group(6))
                p["rounds"] += r
                p["wall"] += float(x.group(5))
                p["idle"] += float(x.group(7))
                p["span"] += span
                p["parents"] += int(x.group(8))
                p["children"] += int(x.group(9))
                if ex:
                    p["fertile"] += int(ex.group(1))
                    p["wide"] += int(ex.group(2))
                pr, ph = phase_of.get(int(x.group(1)), (0, {}))
                for k, v in ph.items():
                    p["phases"][k] += v * pr
            residency[m.group(1)] += 1
        launch, phase_of = [], {}
        continue
    m = RUN.search(line)
    if m:
        if run > 0:
            runs_ms.append(float(m.group(1)))
        run += 1
        print(line)

print(f"\nN={N} M={M} K={K}: {len(runs_ms)} runs after the first: " + ", ".join(f"{x:.1f}" for x in runs_ms) + " ms")
print(f"{'pool':>4} {'rounds':>9} {'period us':>10} {'cycles':>8} {'idle':>6} {'children/parent':>16} {'children/round':>15} "
      f"{'fertile parents':>16} {'wide CTA rounds':>16}")
for h in sorted(pools):
    p = pools[h]
    per = p["wall"] / max(1, p["rounds"])
    print(f"{h:>4} {p['rounds']:>9} {per:>10.4f} {per * a.mhz:>8.0f} {p['idle'] / max(p['span'], 1e-9):>6.1%} "
          f"{p['children'] / max(1, p['parents']):>16.4f} {p['children'] / max(1, p['rounds']):>15.0f} "
          f"{p['fertile'] / max(1, p['parents']):>16.2%} {p['wide']:>16}")
names = list(dict.fromkeys(k for p in pools.values() for k in p["phases"]))  # (in the order of a round)
if names:
    print("\nCTA 0 cycles per round by phase (x: exchange warp)")
    print(f"{'phase':>22} " + " ".join(f"{h:>7}" for h in sorted(pools)))
    for k in names:
        print(f"{k:>22} " + " ".join(f"{pools[h]['phases'][k] / max(1, pools[h]['rounds']):>7.0f}" for h in sorted(pools)))
print("\nresidency (launches):")
for k, v in residency.most_common():
    print(f"  {v:>4} x {k}")

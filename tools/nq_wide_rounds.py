"""Rounds of wide N-Queens device pools (tsb_nq_create_wide, 25-byte records) at the reference's default M = 50 000:
the persistent kernel against two-kernel rounds, and what evaluating each parent's child mask costs the kernel.

  python tools/nq_wide_rounds.py [--M 50000] [--reps 3]

1. us per round, N = 21..24: a pool_run over the whole subtree of each larger golden subtree root
   (tests/golden/nqueens_wide.json) on a warm handle, host clock around the synchronous call, the persistent kernel
   and TSB200_NO_ROUNDS=1 (one tsb_nq_pool_step per round) alternated, `reps` times each; the two routes' counters
   must agree.
2. The phases of a round (TSB200_ROUNDS_PROF: CTA 0's cycles per round) of the same N = 20 subtree on a narrow handle
   (child mask stored in the node) and on a wide one (child mask evaluated when the parents are read), and of the
   N = 21..24 pools.  The parents' child masks are read or evaluated before the profile's "poll-nodes" mark, so the
   difference of those phases is what deriving them costs; the wide node's build and store phases save the child's
   mask evaluation and its packing.
Prints one JSON line per measurement, after the name and power limit of the card."""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200"))
import tsb200  # noqa: E402

GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "nqueens_wide.json")))["subtrees"]
N20_PREFIX = [0, 2, 4, 1, 3]


def subtree_root(N, prefix, wide):
    node = np.zeros(1, dtype=tsb200.NQ_NODE24_DTYPE if wide else tsb200.NQ_NODE_DTYPE)
    b = node["board"][0]
    b[:N] = np.arange(N)
    for d, col in enumerate(prefix):
        j = int(np.nonzero(b[:N] == col)[0][0])
        b[d], b[j] = b[j], b[d]
    node["depth"] = len(prefix)
    return node


def run_subtree(N, prefix, M, wide, no_rounds):
    """the whole subtree in one pool_run call on a handle that has run it once already (its arenas are allocated):
    (seconds, rounds, parents, children, solutions, kernel launches)"""
    if no_rounds:
        os.environ["TSB200_NO_ROUNDS"] = "1"
    else:
        os.environ.pop("TSB200_NO_ROUNDS", None)
    with tsb200.NQueensEvaluator(N, M=M, max_queens=24 if wide else 20) as ev:
        ev.pool_push(subtree_root(N, prefix, wide))
        ev.pool_run(1, M)
        ev.pool_push(subtree_root(N, prefix, wide))
        l0 = ev.kernel_launches
        t0 = time.perf_counter()
        r = ev.pool_run(1, M)
        dt = time.perf_counter() - t0
        return (dt,) + tuple(int(x) for x in r) + (ev.kernel_launches - l0,)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "(nvidia-smi gave no answer)"


PHASES = ["set-up", "poll-nodes", "scan+items", "build", "handoff-wait", "store"]


def profile(N, prefix, M, wide):
    """CTA 0's cycles per round by phase, from the TSB200_ROUNDS_PROF lines of a child process"""
    env = dict(os.environ, TSB200_ROUNDS_PROF="1")
    env.pop("TSB200_NO_ROUNDS", None)
    code = ("import sys; sys.path.insert(0, %r); import nq_wide_rounds as t; t.run_subtree(%d, %r, %d, %r, False)"
            % (os.path.dirname(os.path.abspath(__file__)), N, prefix, M, wide))
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    if p.returncode != 0:
        raise SystemExit(p.stderr)
    rounds, sums = 0, dict.fromkeys(PHASES, 0.0)
    us = []
    for line in p.stderr.splitlines():
        m = re.search(r"LL rounds kernel \(pool 0 of 1\): (\d+) rounds; CTA 0 cycles per round: workers: (.*?) \|", line)
        if m:
            r = int(m.group(1))
            rounds += r
            for ph in PHASES:
                sums[ph] += r * float(re.search(re.escape(ph) + r" ([\d.]+)", m.group(2)).group(1))
        m = re.search(r"LL pace .*?wall ([\d.]+) us, (\d+) rounds", line)
        if m:
            us.append((float(m.group(1)), int(m.group(2))))
    per = {ph: round(sums[ph] / max(1, rounds), 1) for ph in PHASES}
    wall = sum(w for w, _ in us) / max(1, sum(r for _, r in us))
    return {"rounds": rounds, "cycles_per_round": per, "cycles_sum": round(sum(per.values()), 1),
            "us_per_round_in_kernel": round(wall, 3)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--M", type=int, default=50000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    # 1. us per round, the two routes alternated
    for N in (21, 22, 23, 24):
        prefix = [g for g in GOLDEN if g["N"] == N][-1]["prefix"]
        run_subtree(N, prefix, a.M, True, False)  # (warm-up: module load)
        times = {"persistent": [], "two_kernel": []}
        ref = None
        for _ in range(a.reps):
            for route, no_rounds in (("persistent", False), ("two_kernel", True)):
                dt, rounds, parents, children, sols, launches = run_subtree(N, prefix, a.M, True, no_rounds)
                ref = ref or (rounds, parents, children, sols)
                assert (rounds, parents, children, sols) == ref, (route, ref)
                times[route].append((dt, launches))
        rounds = ref[0]
        print(json.dumps({"N": N, "M": a.M, "prefix": prefix, "rounds": rounds, "tree": ref[2], "sol": ref[3],
                          **{f"us_per_round_{k}": [round(1e6 * dt / rounds, 2) for dt, _ in v] for k, v in times.items()},
                          **{f"launches_{k}": v[0][1] for k, v in times.items()}}), flush=True)
    # 2. the phases of a round: N = 20 narrow against N = 20 wide (same nodes), then N = 21..24
    for N, prefix, wide in [(20, N20_PREFIX, False), (20, N20_PREFIX, True)] + \
            [(N, [g for g in GOLDEN if g["N"] == N][-1]["prefix"], True) for N in (21, 22, 23, 24)]:
        for rep in range(a.reps):
            print(json.dumps({"profile": {"N": N, "wide": wide, "rep": rep, "M": a.M, **profile(N, prefix, a.M, wide)}}),
                  flush=True)


if __name__ == "__main__":
    main()

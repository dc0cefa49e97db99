"""The PFSP offload loop at the reference's default --M 50000 (and any M given): tsb_pfsp_pool_run through the persistent kernel
(csrc/pfsp_rounds.cuh) against the loop of tsb_pfsp_pool_step (the same call with TSB200_NO_ROUNDS=1), alternately on
identical start pools (the root's 380 grandchildren, incumbent = the optimum, as under --ub 1).  Prints the card, its
power limit, the rounds, the microseconds per round of every run (synchronised wall clock: pool_run returns after its
last round) and whether the two routes' counters and drained pools are identical.

    python tools/pfsp_rounds.py [runs [M ...]]  (default 3 runs, M = 50000; ta020 only at M = 50000;
                                                 TSB200_ROUNDS_PROF=1: the kernel's phase counters on stderr)
"""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                "gpu-accelerated-tree-search-chapel_b200"))
import tsb200  # noqa: E402

OPT = {14: 1377, 20: 1591}
CONFIGS = [(14, "lb1"), (14, "lb1_d"), (20, "lb1_d")]
m = 25


def start_pool(jobs=20):
    nodes = np.zeros(jobs * (jobs - 1), dtype=tsb200.PFSP_NODE_DTYPE)
    x = 0
    for i in range(jobs):
        for j in range(1, jobs):
            prmu = np.arange(jobs)
            prmu[[0, i]] = prmu[[i, 0]]
            prmu[[1, j]] = prmu[[j, 1]]
            nodes["prmu"][x, :jobs] = prmu
            x += 1
    nodes["depth"], nodes["limit1"] = 2, 1
    return nodes


def one(ev, inst, lb, M, steps):
    if steps:
        os.environ["TSB200_NO_ROUNDS"] = "1"
    else:
        os.environ.pop("TSB200_NO_ROUNDS", None)
    ev.pool_push(start_pool())
    l0 = ev.kernel_launches
    t0 = time.perf_counter()
    res = ev.pool_run(lb, m, M, OPT[inst])
    dt = time.perf_counter() - t0
    return res, dt, ev.kernel_launches - l0, ev.pool_drain()


def main():
    runs = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    Ms = [int(x) for x in sys.argv[2:]] or [50000]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    for M, inst, lb in [(M, inst, lb) for M in Ms for inst, lb in CONFIGS if inst == 14 or M == 50000]:
        with tsb200.PfspEvaluator(inst, M=M) as ev:
            one(ev, inst, lb, M, False)  # warm-up: module load, arena, side arrays
            one(ev, inst, lb, M, True)
            times = {False: [], True: []}
            outs = {}
            for _ in range(runs):
                for steps in (True, False):
                    res, dt, launches, rest = one(ev, inst, lb, M, steps)
                    times[steps].append(dt)
                    outs.setdefault(steps, (res, launches, rest.tobytes()))
                    assert outs[steps][0] == res and outs[steps][2] == rest.tobytes()
            (rs, ls, ps), (rp, lp, pp) = outs[True], outs[False]
            rounds = rs[0]
            us = {k: sorted(1e6 * t / max(1, rounds) for t in v) for k, v in times.items()}
            print(f"ta{inst:03d} {lb} M={M}: rounds {rounds}, parents {rs[1]}, children {rs[2]}, solutions {rs[3]}, "
                  f"best {rs[4]}; launches step loop {ls}, persistent {lp}")
            print(f"  us per round: step loop {', '.join(f'{x:.2f}' for x in us[True])}; "
                  f"persistent {', '.join(f'{x:.2f}' for x in us[False])}")
            print(f"  identical counters: {rs == rp}; identical drained pools: {ps == pp}")
    os.environ.pop("TSB200_NO_ROUNDS", None)


if __name__ == "__main__":
    main()

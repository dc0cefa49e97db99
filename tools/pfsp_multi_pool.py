"""Several PFSP device pools in one launch of the persistent kernel (tsb_pfsp_pool_run_multi) against the same pools
run one after the other (tsb_pfsp_pool_run per pool), alternately on identical start pools: the root's 380
grandchildren (tools/pfsp_rounds.py), split strided into K pools (the reference's static split), incumbent = the
optimum (as under --ub 1), each pool run to exhaustion.  Prints the card, its power limit and max SM clock, every
run's wall time (synchronised: both calls return after their last round) and microseconds per pool-round (wall time
over the rounds of all K pools), and whether the two ways' counters and drained pools are identical.

    python tools/pfsp_multi_pool.py [runs [M ...]]   (default 3 runs; M = 300 6000 20000 25000 50000, the last for
                                                      K <= 2 only, the K-pool capacity on an H100 being 25 344 for
                                                      K = 4; ta020 only from M = 20 000: below that its 860 M-node tree
                                                      takes more than a second per run)
"""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pfsp_rounds import OPT, start_pool  # noqa: E402  (also puts the package on sys.path)

import tsb200  # noqa: E402

CONFIGS = [(14, "lb1"), (14, "lb1_d"), (20, "lb1_d")]
m = 25


def split(K):
    s = start_pool()
    return [np.ascontiguousarray(s[i::K]) for i in range(K)]


def one(evs, inst, lb, M, multi):
    for ev, s in zip(evs, split(len(evs))):
        ev.pool_push(s)
    t0 = time.perf_counter()
    if multi:
        res = tsb200.pfsp_pool_run_multi(evs, lb, m, M, [OPT[inst]] * len(evs))
    else:
        res = [ev.pool_run(lb, m, M, OPT[inst]) for ev in evs]
    dt = time.perf_counter() - t0
    return res, dt, b"".join(ev.pool_drain().tobytes() for ev in evs)


def main():
    runs = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    Ms = [int(x) for x in sys.argv[2:]] or [300, 6000, 20000, 25000, 50000]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}; SMs: {tsb200.lib().tsb_device_sm_count(0)}")
    for inst, lb in CONFIGS:
        for M in Ms:
            if inst == 20 and M < 20000:
                continue
            with tsb200.PfspEvaluator(inst, M=M) as ev:
                for K in (1, 2, 3, 4):
                    if M == 50000 and K > 2:
                        continue
                    evs = [ev] + [ev.sibling(i) for i in range(1, K)]
                    shared = ev.pools_per_launch(lb, M) >= K
                    one(evs, inst, lb, M, True)  # warm-up: module load, arenas
                    one(evs, inst, lb, M, False)
                    times, outs = {True: [], False: []}, {}
                    for _ in range(runs):
                        for multi in (False, True):
                            res, dt, rest = one(evs, inst, lb, M, multi)
                            times[multi].append(dt)
                            outs.setdefault(multi, (res, rest))
                            assert outs[multi] == (res, rest)
                    (rs, ps), (rm, pm) = outs[False], outs[True]
                    rounds = sum(r[0] for r in rs)
                    us = {k: [1e6 * t / max(1, rounds) for t in v] for k, v in times.items()}
                    print(f"ta{inst:03d} {lb} M={M} K={K} ({'one launch' if shared else 'one after the other'}): "
                          f"pool-rounds {rounds} ({', '.join(str(r[0]) for r in rs)}), children {sum(r[2] for r in rs)}")
                    for k, name in ((False, "pool_run x K"), (True, "pool_run_multi")):
                        print(f"  {name}: wall ms {', '.join(f'{1e3 * t:.2f}' for t in times[k])}; "
                              f"us per pool-round {', '.join(f'{x:.2f}' for x in us[k])}")
                    print(f"  identical counters: {rs == rm}; identical drained pools: {ps == pm}")
                    sys.stdout.flush()


if __name__ == "__main__":
    main()

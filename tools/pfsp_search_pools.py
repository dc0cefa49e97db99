"""Whole PFSP searches with K device pools on one GPU (tsb_pfsp_search_on_pools) against the one-pool search
(tsb_pfsp_search_on), on handles created (with their siblings) before any timing, alternately K = 1, 2, 3, 4 per
repetition: ub = 1, m = 25, D = 1.  Prints the card, its power limit and max SM clock, then per workload and K the
step-2 seconds of every run (the device part of the search; steps 1 and 3 are the host's), the counts (tree, sol,
best must equal K = 1's), offloads and kernel launches.

    python tools/pfsp_search_pools.py [runs]   (default 3)
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200"))

import tsb200  # noqa: E402

# ta014 lb1 and ta020 lb1_d (Chapel min_heads: 17 192 rounds at M = 50 000) at the reference's default M, where two
# pools share a launch on an H100; ta020 lb2, whose pools always run one after the other
WORKLOADS = [(14, "lb1", 50000), (20, "lb1_d", 50000), (20, "lb2", 50000)]


def main():
    runs = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}; SMs: {tsb200.lib().tsb_device_sm_count(0)}")
    for inst, lb, M in WORKLOADS:
        with tsb200.PfspEvaluator(inst, M=M) as ev:
            for i in range(1, 4):
                ev.sibling(i)
            ev.search(inst, lb, 1, 25, M, pools=2)  # warm-up: module load, arenas of two pools
            t2, stats = {K: [] for K in (1, 2, 3, 4)}, {}
            for _ in range(runs):
                for K in (1, 2, 3, 4):
                    st = ev.search(inst, lb, 1, 25, M, pools=K)
                    t2[K].append(st.t_step2)
                    stats[K] = st
            base = stats[1]
            for K in (1, 2, 3, 4):
                st = stats[K]
                same = (st.explored_tree, st.explored_sol, st.best) == (base.explored_tree, base.explored_sol, base.best)
                print(f"ta{inst:03d} {lb} M={M} K={K} ({ev.pools_per_launch(lb, M)} pools per launch): step 2 s "
                      f"{', '.join(f'{x:.4f}' for x in t2[K])}; best of K=1 / best of K: "
                      f"{min(t2[1]) / min(t2[K]):.2f}x; tree {st.explored_tree} sol {st.explored_sol} best {st.best} "
                      f"(same as K=1: {same}); offloads {st.offloads}, launches {st.kernel_launches}")
                sys.stdout.flush()


if __name__ == "__main__":
    main()

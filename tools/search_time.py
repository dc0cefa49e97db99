#!/usr/bin/env python
"""Wall time of whole device-pool searches: python tools/search_time.py N M [reps [D]]   (env knobs apply, e.g. TSB200_POOLS=1)"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200")]
import tsb200  # noqa: E402

N, M = int(sys.argv[1]), int(sys.argv[2])
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
D = int(sys.argv[4]) if len(sys.argv) > 4 else 1
tsb200.nqueens_search_device(min(N, 12), 1, 25, M, 1)
ev = tsb200.NQueensEvaluator(N, M=M) if D == 0 else None  # D = 0: on a handle created once (as bench.py's e2e leg)
if ev is not None:
    ev.search(25, M)
    D = 1
for r in range(reps):
    t0 = time.perf_counter()
    st = ev.search(25, M) if ev is not None else tsb200.nqueens_search_device(N, 1, 25, M, D)
    dt = time.perf_counter() - t0
    print(f"N={N} M={M} D={D}: steals {st.steals} shares {[round(x / max(1, st.explored_tree), 3) for x in st.per_gpu_tree[:D]]} tree {st.explored_tree} sol {st.explored_sol} offloads {st.offloads} launches {st.kernel_launches} "
          f"{dt * 1e3:.1f} ms  {st.explored_tree / dt / 1e9:.2f} Gnodes/s", flush=True)

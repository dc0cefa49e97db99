"""The whole search of a board of 21 to 24 queens (default N = 21) on the GPU(s), as a `-sMAX_QUEENS=24` build of the
reference runs it: the 3-step search with the pool of step 2 resident on the device (tsb_nq_search_device, 25-byte
nodes, one device pool per task).  Chunks of up to the one-pool capacity of the persistent kernel (67 584 parents on
an H100; the reference's default is --M 50000) run the whole offload loop in that kernel, larger ones (the default
here) two kernels per round.  Prints the explored tree, the solutions against the published count (OEIS A000170), the
time, and the name and power limit of every card the search used; exits 1 when the solution count differs.

  python tools/nq_wide_search.py [--N 21] [--M 4194304] [--D 1] [--host]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200"))
import tsb200  # noqa: E402

SOLUTIONS = json.load(open(os.path.join(ROOT, "tests", "golden", "nqueens_wide.json")))["solutions_oeis_a000170"]


def cards(D):
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    lines = q.stdout.strip().splitlines() if q.returncode == 0 else []
    return lines[:D] if lines else ["(nvidia-smi gave no answer)"]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--N", type=int, default=21)
    ap.add_argument("--m", type=int, default=25)
    ap.add_argument("--M", type=int, default=4194304)
    ap.add_argument("--D", type=int, default=1)
    ap.add_argument("--host", action="store_true", help="the host-pool search (tsb_nq_search) instead")
    a = ap.parse_args()
    if not 21 <= a.N <= 24:
        ap.error("--N must be 21..24")
    for c in cards(a.D):
        print("card:", c, flush=True)
    t0 = time.time()
    search = tsb200.nqueens_search if a.host else tsb200.nqueens_search_device
    st = search(a.N, 1, a.m, a.M, a.D)
    wall = time.time() - t0
    steps = st.t_step1 + st.t_step2 + st.t_step3
    want = SOLUTIONS[str(a.N)]
    print(json.dumps({
        "N": a.N, "m": a.m, "M": a.M, "D": a.D, "route": "host pool" if a.host else "device pool",
        "explored_tree": st.explored_tree, "explored_sol": st.explored_sol, "published_sol": want,
        "seconds_steps": round(steps, 3), "seconds_wall": round(wall, 3),
        "gnodes_per_s": round(st.explored_tree / steps / 1e9, 3), "offloads": st.offloads,
        "kernel_launches": st.kernel_launches}), flush=True)
    if st.explored_sol != want:
        print(f"solution count {st.explored_sol} != {want}", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())

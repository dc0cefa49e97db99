"""The whole search of a board of 21 to 24 queens (default N = 21) on the GPU(s), as a `-sMAX_QUEENS=24` build of the
reference runs it: the 3-step search with the pool of step 2 resident on the device (tsb_nq_search_device, 25-byte
nodes, one device pool per task).  Chunks of up to the one-pool capacity of the persistent kernel (67 584 parents on
an H100; the reference's default is --M 50000) run the whole offload loop in that kernel, larger ones (the default
here) two kernels per round.  Prints the explored tree, the solutions against the published count (OEIS A000170), the
time, and the name and power limit of every card the search used; exits 1 when the solution count differs.
--checkpoint FILE makes the search resumable (tsb_nq_search_device_ckpt): it stops after --time-limit seconds or on
SIGINT / SIGTERM, writes FILE, prints the counts so far and exits 4; the same command continues it from FILE, so a
search of hours runs in slots.  The printed stats are then those of the whole search over every run.

  python tools/nq_wide_search.py [--N 21] [--M 4194304] [--D 1] [--host] [--checkpoint FILE [--time-limit S]]
"""
import argparse
import json
import os
import signal
import subprocess
import sys
import threading
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
    ap.add_argument("--checkpoint", default=None, help="resumable search: continue from / stop into this file")
    ap.add_argument("--time-limit", type=float, default=None, help="seconds of this run before it stops")
    a = ap.parse_args()
    if not 21 <= a.N <= 24:
        ap.error("--N must be 21..24")
    if (a.checkpoint or a.time_limit is not None) and (a.host or not a.checkpoint):
        ap.error("--checkpoint needs the device-pool search, and --time-limit needs --checkpoint")
    for c in cards(a.D):
        print("card:", c, flush=True)
    t0 = time.time()
    if a.checkpoint:
        # the search runs in a thread, so that this (main) thread takes SIGINT / SIGTERM while it runs
        for sig in (signal.SIGINT, signal.SIGTERM):
            signal.signal(sig, lambda *_: tsb200.request_stop())
        done = {}

        def run():
            try:
                done["st"] = tsb200.nqueens_search_device(a.N, 1, a.m, a.M, a.D, checkpoint=a.checkpoint,
                                                          time_limit=a.time_limit)
            except tsb200.TsbError as e:
                done["error"] = e
        th = threading.Thread(target=run)
        th.start()
        while th.is_alive():
            th.join(0.5)
        e = done.get("error")
        if e is not None and not isinstance(e, tsb200.SearchStopped):
            raise e
        if e is not None:
            print(json.dumps({"N": a.N, "m": a.m, "M": a.M, "D": a.D, "stopped": True, "checkpoint": a.checkpoint,
                              "explored_tree_so_far": e.stats.explored_tree, "explored_sol_so_far": e.stats.explored_sol,
                              "seconds_step2_so_far": round(e.stats.t_step2, 3),
                              "seconds_wall": round(time.time() - t0, 3)}), flush=True)
            print(f"checkpoint written to {a.checkpoint}; rerun the same command to resume", file=sys.stderr)
            return 4
        st = done["st"]
    else:
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

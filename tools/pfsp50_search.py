#!/usr/bin/env python
"""Speed of a 50-job PFSP search (ta031..ta060, a MAX_JOBS = 50 build) on device pools: the resumable search
(tsb_pfsp_search_device_ckpt_wide) stopped after --seconds, --runs times, reporting explored nodes per second of step 2
(Mnodes/s) and rounds per second.  --host: the host-pool search instead (tsb_pfsp_search_ckpt_wide: the pool stays on
the CPU, every chunk is one tsb_pfsp_evaluate; "rounds" are then offloads, and --pools does not apply).  Each run
starts from scratch (its checkpoint lives in a temporary directory), so runs are independent and alternate with
nothing else; a run that stops reports its checkpoint's size (TSB200_TRACE=1 also prints the time taken to write it).
Prints the card's name, power limit and SM clock first.

  python tools/pfsp50_search.py --inst 31 --lb lb1 --ub 1 --M 50000 --seconds 20 --runs 3
  TSB200_TRACE=1 python tools/pfsp50_search.py --host --inst 31 --lb lb1 --ub 1 --M 50000 --seconds 5 --runs 2
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200"))
import tsb200  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inst", type=int, default=31)
    ap.add_argument("--lb", default="lb1")
    ap.add_argument("--ub", type=int, default=1)
    ap.add_argument("--m", type=int, default=25)
    ap.add_argument("--M", type=int, default=50000)
    ap.add_argument("--D", type=int, default=1)
    ap.add_argument("--pools", type=int, default=1)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--host", action="store_true", help="the host-pool search (tsb_pfsp_search_ckpt_wide)")
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("gpu:", smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else "unknown")
    for run in range(a.runs):
        with tempfile.TemporaryDirectory() as tmp:
            ck = os.path.join(tmp, "ck")
            try:
                if a.host:
                    st = tsb200.pfsp_search_wide(a.inst, a.lb, a.ub, a.m, a.M, a.D, checkpoint=ck, time_limit=a.seconds)
                else:
                    st = tsb200.pfsp_search_device_wide(a.inst, a.lb, a.ub, a.m, a.M, a.D, a.pools, checkpoint=ck,
                                                        time_limit=a.seconds)
                finished = True
            except tsb200.SearchStopped as e:
                st, finished = e.stats, False
            ck_bytes = os.path.getsize(ck) if os.path.exists(ck) else 0
        t2 = max(st.t_step2, 1e-9)
        print(json.dumps({"run": run, "pool": "host" if a.host else "device", "inst": a.inst, "lb": a.lb, "ub": a.ub,
                          "M": a.M, "D": a.D, "pools": None if a.host else a.pools, "finished": finished,
                          "checkpoint_bytes": ck_bytes, "tree": st.explored_tree, "sol": st.explored_sol, "best": st.best,
                          "rounds": st.offloads, "t_step2": round(t2, 3), "Mnodes_per_s": round(st.explored_tree / t2 / 1e6, 3),
                          "rounds_per_s": round(st.offloads / t2, 1)}), flush=True)


if __name__ == "__main__":
    main()

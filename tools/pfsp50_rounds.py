"""50-job PFSP device pools (ta031..ta060): the persistent kernel (csrc/pfsp_wide_rounds.cuh) against the step loop of
two-kernel rounds (the same call under TSB200_NO_ROUNDS=1), alternately on identical start pools.

A workload is one library call of the resumable device-pool search (tsb_pfsp_search_device_ckpt_wide, D = 1, K pools,
m = 25, --ub 1: best = the optimum): step 1 expands the root breadth-first until the pool holds 25 K nodes (the root's
children, or some grandchildren), the reference's strided split gives the K start pools, one call runs 1024 rounds of
one pool (K = 1) or 256 rounds of each of K pools (K > 1: the search's own cadence, which rebalances the pools between
calls), and the search stops with a checkpoint.  Per (instance, K): one warm-up call of each route; then per M three
alternations.  Prints the card, its power limit and max SM clock, every run's microseconds per pool-round (the time
inside the library's pool calls, from the search's TSB200_TRACE line: no handle set-up, pool push, drain or checkpoint)
and whether the two routes leave identical checkpoints (every field but the times and kernel_launches).

The round split: for K = 1, one more step-loop call under torch.profiler gives the device time of its two kernels per
round against the time per round; the rest is launch, host wait and host bookkeeping.

    python tools/pfsp50_rounds.py [--runs 3] [--inst 31 41 51] [--K 1 2 3 4] [--M M ...]
        (--M: chunk sizes instead of the default list; "cap" and "cap+1" stand for the K-pool capacity edges;
         TSB200_ROUNDS_PROF=1: the kernel's phase counters on stderr)
"""
import argparse
import os
import re
import shutil
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                "gpu-accelerated-tree-search-chapel_b200"))
import tsb200  # noqa: E402

CONFIGS = [(31, "lb1"), (41, "lb1_d"), (51, "lb1")]
m = 25
# checkpoint fields that differ between routes or runs: t_step1, t_step2; the task's kernel_launches; the checksum
TIMES, LAUNCHES = slice(72, 88), slice(128, 136)
TRACE = re.compile(rb"\[tsb200\] task 0: (\d+) pools, (\d+) rounds in ([0-9.]+) ms of pool calls")


def capacities():
    sms = tsb200.lib().tsb_device_sm_count(0)
    return {K: min(sms if K == 1 else 2 * sms // K, 256) * 384 for K in (1, 2, 3, 4)}


def chunk_sizes(K, cap, Ms):
    """by default M = 1 000, 6 000, 20 000 and the capacity edges of K pools (for K <= 2 the edges 50 688 / 50 689
    stand for the reference's default 50 000)"""
    edge = {"cap": cap[K], "cap+1": cap[K] + 1}
    return sorted({edge[x] if x in edge else int(x) for x in Ms})


def one(path, log, inst, lb, K, M, kernel):
    """(rounds, microseconds per pool-round, what the call left: the checkpoint without times and launches)"""
    if kernel:
        os.environ.pop("TSB200_NO_ROUNDS", None)
    else:
        os.environ["TSB200_NO_ROUNDS"] = "1"
    if os.path.exists(path):
        os.remove(path)
    saved = os.dup(2)  # the library's stderr -> log
    with open(log, "wb") as f:
        os.dup2(f.fileno(), 2)
    try:
        st = tsb200.pfsp_search_device_wide(inst, lb, 1, m, M, 1, K, checkpoint=path, time_limit=0.0)
        key = ("finished", st.explored_tree, st.explored_sol, st.best, st.offloads, st.offloaded_parents)
    except tsb200.SearchStopped:
        b = bytearray(open(path, "rb").read())
        b[TIMES] = bytes(16)
        b[LAUNCHES] = bytes(8)
        key = bytes(b[:-8])
    finally:
        os.dup2(saved, 2)
        os.close(saved)
        os.environ.pop("TSB200_NO_ROUNDS", None)
    hit = TRACE.search(open(log, "rb").read())
    rounds, ms = int(hit.group(2)), float(hit.group(3))
    return rounds, 1e3 * ms / max(1, rounds), key


def kernel_split(path, log, inst, lb, M):
    """device time of the step loop's kernels per round, from torch.profiler (None: no kernel was recorded)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rounds, us, _ = one(path, log, inst, lb, 1, M, False)
    dev = sum(e.device_time_total for e in prof.key_averages() if "pfsp_wide_expand" in e.key)
    return (dev / max(1, rounds) if dev else None), us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--inst", type=int, nargs="+", default=[c[0] for c in CONFIGS])
    ap.add_argument("--K", type=int, nargs="+", default=[1, 2, 3, 4])
    ap.add_argument("--M", nargs="+", default=["1000", "6000", "20000", "cap", "cap+1"])
    a = ap.parse_args()
    runs = a.runs
    os.environ["TSB200_TRACE"] = "1"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    cap = capacities()
    print(f"card: {card}; SMs: {tsb200.lib().tsb_device_sm_count(0)}; pool capacities K=1..4: "
          f"{', '.join(str(cap[K]) for K in (1, 2, 3, 4))}")
    # (a checkpoint holds every node of the pools: up to GBs; in memory where there is room)
    shm = "/dev/shm" if os.path.isdir("/dev/shm") and shutil.disk_usage("/dev/shm").free > 24 << 30 else None
    tmp = tempfile.mkdtemp(prefix="pfsp50_rounds_", dir=shm)
    path, log = os.path.join(tmp, "ck"), os.path.join(tmp, "log")
    try:
        for inst, lb in [c for c in CONFIGS if c[0] in a.inst]:
            for K in a.K:
                one(path, log, inst, lb, K, 1000, True)  # warm-up: module load, first launches
                one(path, log, inst, lb, K, 1000, False)
                for M in chunk_sizes(K, cap, a.M):
                    us, outs = {True: [], False: []}, {}
                    for _ in range(runs):
                        for kernel in (False, True):
                            rounds, x, key = one(path, log, inst, lb, K, M, kernel)
                            us[kernel].append(x)
                            outs.setdefault(kernel, key)
                            assert outs[kernel] == key, "a route is not deterministic"
                    print(f"ta{inst:03d} {lb} K={K} M={M}: pool-rounds {rounds}; us per pool-round: step loop "
                          f"{', '.join(f'{x:.1f}' for x in us[False])}; kernel {', '.join(f'{x:.1f}' for x in us[True])}; "
                          f"identical: {outs[True] == outs[False]}")
                    if K == 1 and inst == 31:
                        kt, wall = kernel_split(path, log, inst, lb, M)
                        print("  step-loop split: " + (f"kernels {kt:.1f} us of {wall:.1f} us per round" if kt else
                                                       "not measured (no kernel in the profile)"))
                    sys.stdout.flush()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Pin whole PFSP searches whose counts depend on how the incumbent `best` moves: ub = 0 (best starts at the int64
maximum and falls as leaves are found), lb2 (its early exit reads best), per-task incumbents of the D-way split and
the parts of a process-per-GPU launch.

Source of the values: the CPU oracle (oracle/tsb_oracle.c, a restatement of the reference's Chapel drivers with the
oracle as evaluator):
  * or_pfsp_search_offload(inst, lb, ub, m, M, D): the 3-step search of pfsp_gpu_chpl.chpl:306-431 (D = 1) and
    pfsp_multigpu_chpl.chpl:316-560 (D > 1: static strided split, per-task best_l from best, min reduce, no
    stealing) -> tree, sol, best, offloads, offloaded_parents and, per task, its step-2 tree / sol / final best_l;
  * or_pfsp_search_offload_part(..., part): task `part` of that split run alone, step 1 credited to part 0, step 3
    on its own leftovers with its own best.
One entry serves the host-pool and the device-pool searches of the library: both follow this chunk sequence.

    make -C oracle && python tests/golden/make_golden_searches.py        (CPU only; the entries run in parallel)

Oracle time per entry on one core of an x86 build host (gcc -O2), the entries running side by side: ta014 lb2 ub 0
M 50 000: 245 s; M 700: 55 s; M 3000 D 3: 238 s; lb1 ub 1 M 3000 D 3: 6.4 s, its parts 4.0 / 1.3 / 1.6 s.
"""
import json
import os
import sys
from concurrent.futures import ProcessPoolExecutor, as_completed

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pyoracle as po  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pfsp_searches.json")
LB = {"lb1_d": 0, "lb1": 1, "lb2": 2}
M_SMALL = 25  # m

# (inst, lb, ub, M, D, with_parts)
CONFIGS = [
    (14, "lb2", 0, 50000, 1, False),
    (14, "lb2", 0, 700, 1, False),    # many small rounds, many of them redone by the sequential rule
    (14, "lb2", 0, 3000, 3, False),
    (14, "lb1", 1, 3000, 3, True),
]
# Not pinned: ub = 0 searches of lb1 / lb1_d with D > 1 (ta014 lb1 M 50 000 D 4, lb1_d M 300 D 2, lb1_d M 50 000 D 2
# and its parts): each task starts step 2 with no incumbent of its own, and the oracle had not finished any of them
# after ten minutes.


def key(inst, lb, ub, M, D):
    return f"ta{inst:03d}_{lb}_ub{ub}_M{M}_D{D}"


def counts(r, D):
    return {"tree": r.tree, "sol": r.sol, "best": r.best, "offloads": r.offloads,
            "offloaded_parents": r.offloaded_parents, "task_tree": list(r.task_tree[:D]),
            "task_sol": list(r.task_sol[:D]), "task_best": list(r.task_best[:D])}


def run(job):
    inst, lb, ub, M, D, part = job
    if part is None:
        r = po.pfsp_search_offload(inst, LB[lb], ub, M_SMALL, M, D)
    else:
        r = po.pfsp_search_offload_part(inst, LB[lb], ub, M_SMALL, M, D, part)
    return job, counts(r, D), r.seconds


def main():
    jobs = []
    for inst, lb, ub, M, D, with_parts in CONFIGS:
        jobs.append((inst, lb, ub, M, D, None))
        if with_parts:
            jobs += [(inst, lb, ub, M, D, p) for p in range(D)]
    # the slow lb2 entries first, so that they overlap
    jobs.sort(key=lambda j: j[1] != "lb2")
    done = {}
    with ProcessPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1)) as ex:
        for f in as_completed([ex.submit(run, j) for j in jobs]):
            j, c, s = f.result()
            done[j] = (c, s)
            print(f"{j}: {s:.1f} s", file=sys.stderr, flush=True)
    out = {"_source": "oracle/tsb_oracle.c: or_pfsp_search_offload(inst, lb, ub, m = 25, M, D) for each entry; "
                      "'parts': or_pfsp_search_offload_part(..., part) for every part (tests/golden/"
                      "make_golden_searches.py)",
           "m": M_SMALL, "searches": {}}
    for inst, lb, ub, M, D, with_parts in CONFIGS:
        e = {"inst": inst, "lb": lb, "ub": ub, "M": M, "D": D}
        e.update(done[(inst, lb, ub, M, D, None)][0])
        if with_parts:
            e["parts"] = [done[(inst, lb, ub, M, D, p)][0] for p in range(D)]
        out["searches"][key(inst, lb, ub, M, D)] = e
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()

"""Whole PFSP searches of a MAX_JOBS = 50 build (ta031..ta060) on host pools and device pools, against the reference:

- the tree, solution and optimum counts of the reference's own C program built with MAX_JOBS = 50 under --ub 1
  (tests/golden/pfsp50_searches.json, tests/golden/make_golden_pfsp50.py), with m = 1 (the root goes to the GPU) and
  m = 25, D = 1 and 2, one and two device pools per task;
- round by round, on searches that do not finish: the resumable search stopped after its first library call (1024
  rounds) leaves a checkpoint whose pool (in order), counters and incumbent are those of the reference's pool loop run
  for as many rounds by the oracle built with OR_MAX_JOBS = 50 (or_pfsp_expand_chunk: evaluate + the sequential
  generate_children of pfsp_gpu_chpl.chpl).  ub = 0 reaches leaves, so rounds in which a leaf lowers the incumbent
  inside the chunk (the library's slow path) are among those compared; a tiny arena covers compaction and growth;
- a search stopped and resumed several times equals the same prefix of one uninterrupted pool loop after every call."""
import ctypes as C
import json
import os
import struct
from collections import deque

import numpy as np
import pytest

import tsb200
from oracle import pyoracle50 as po50

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "pfsp50_searches.json")))["searches"]
REC = 208
ROUNDS_PER_CALL = 1024
LB = {"lb1_d": 0, "lb1": 1, "lb2": 2}


def golden(key):
    g = GOLDEN[key]
    return g["tree"], g["sol"], g["best"]


@pytest.mark.parametrize("m", [1, 25])
@pytest.mark.parametrize("key", sorted(GOLDEN))
def test_host_pool_search_matches_reference(key, m):
    inst, lb = int(key[2:5]), key[6:]
    for D in (1, 2):
        st = tsb200.pfsp_search_wide(inst, lb, 1, m, 50000, D)
        assert (st.explored_tree, st.explored_sol, st.best) == golden(key), (D, st.explored_tree)


@pytest.mark.parametrize("m", [1, 25])
@pytest.mark.parametrize("key", sorted(GOLDEN))
def test_device_pool_search_matches_reference(key, m):
    inst, lb = int(key[2:5]), key[6:]
    for D in (1, 2):
        for pools in (1, 2):
            st = tsb200.pfsp_search_device_wide(inst, lb, 1, m, 50000, D, pools)
            assert (st.explored_tree, st.explored_sol, st.best) == golden(key), (D, pools, st.explored_tree)
            if m == 1 and D * pools == 1:  # (the root itself goes to the device pool)
                assert st.offloads > 0 and st.kernel_launches > 0


# ---------------------------------------------------------------------------------------------- the oracle's pool loop
def root():
    r = np.zeros(1, dtype=po50.PFSP_NODE_DTYPE)
    r["limit1"] = -1
    r["prmu"][0] = np.arange(50)
    return r


def expand(t, lb, parents, best):
    """or_pfsp_expand_chunk: the children (reference order), the leaves and the incumbent after the chunk"""
    L = po50.lib()
    L.or_pfsp_expand_chunk.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int64), C.c_void_p,
                                       C.c_int64, C.POINTER(C.c_uint64)]
    L.or_pfsp_expand_chunk.restype = C.c_int64
    parents = np.ascontiguousarray(parents)
    out = np.zeros(max(1, len(parents) * 50), dtype=po50.PFSP_NODE_DTYPE)
    b, sol = C.c_int64(best), C.c_uint64(0)
    n = L.or_pfsp_expand_chunk(C.byref(t), lb, parents.ctypes.data, len(parents), C.byref(b), out.ctypes.data,
                               len(out), C.byref(sol))
    assert n >= 0
    return out[:n], int(sol.value), int(b.value)


def oracle_search(inst, lb, ub, m, M, calls):
    """step 1 (breadth first until the pool holds m nodes) and the step-2 state after each of `calls` blocks of
    ROUNDS_PER_CALL rounds of popBackBulk(m, M) + expand; plus how many rounds lowered the incumbent inside the chunk"""
    t = po50.tables(inst)
    best = int(tsb200.lib().tsb_taillard_best_ub(inst)) if ub else 2**63 - 1
    tree1 = sol1 = 0
    q = deque([root()[0]])
    while len(q) < m and q:
        kids, s, best = expand(t, lb, np.array([q.popleft()], dtype=po50.PFSP_NODE_DTYPE), best)
        tree1 += len(kids)
        sol1 += s
        q.extend(kids)
    step1 = (tree1, sol1, best)
    buf = np.array(list(q), dtype=po50.PFSP_NODE_DTYPE)  # the pool is buf[:size], a stack
    size = len(buf)
    tree = sol = offloads = parents = improved = 0
    snaps = []
    for _ in range(calls):
        for _ in range(ROUNDS_PER_CALL):
            if size < m:
                break
            n = min(size, M)
            size -= n
            kids, s, nb = expand(t, lb, buf[size:size + n], best)
            improved += nb < best
            best = nb
            if size + len(kids) > len(buf):
                buf = np.concatenate([buf[:size], np.zeros(max(len(buf), len(kids)), dtype=buf.dtype)])
            buf[size:size + len(kids)] = kids
            size += len(kids)
            tree += len(kids)
            sol += s
            offloads += 1
            parents += n
        snaps.append(dict(tree=tree, sol=sol, offloads=offloads, parents=parents, best=best, pool=buf[:size].tobytes()))
    return step1, snaps, improved


def read_ckpt(path):
    """the fields of a one-task, one-pool checkpoint (layout: csrc/search_ckpt.cpp)"""
    b = open(path, "rb").read()
    assert b[:8] == b"TSB200CK"
    version, problem, rec = struct.unpack_from("<3I", b, 8)
    assert (version, problem, rec) == (1, 2, REC)
    o = 20 + 7 * 4
    tree1, sol1, best1 = struct.unpack_from("<QQq", b, o)
    o += 24 + 16 + 8
    tree, sol, offloads, parents, launches, best, finished, pools, left = struct.unpack_from("<5Qq2IQ", b, o)
    o += 5 * 8 + 8 + 8 + 8
    assert finished == 0 and pools == 1 and left == 0
    pbest, count = struct.unpack_from("<qQ", b, o)
    o += 16
    nodes = b[o:o + count * REC]
    return (tree1, sol1, best1), dict(tree=tree, sol=sol, offloads=offloads, parents=parents, best=pbest, pool=nodes)


def stop_after_one_call(path, inst, lb, ub, m, M):
    with pytest.raises(tsb200.SearchStopped):
        tsb200.pfsp_search_device_wide(inst, lb, ub, m, M, 1, 1, checkpoint=str(path), time_limit=0.0)
    return read_ckpt(path)


def compare(got, want):
    assert {k: got[k] for k in ("tree", "sol", "offloads", "parents", "best")} == \
        {k: want[k] for k in ("tree", "sol", "offloads", "parents", "best")}
    assert got["pool"] == want["pool"], f"pools differ ({len(got['pool']) // REC} vs {len(want['pool']) // REC} nodes)"


# (lb1_d under ub = 1 prunes these instances to a search that ends inside the first call: it has no checkpoint to
# compare, and the golden counts cover it)
PARITY = [(inst, lb, ub, M) for inst in (31, 41, 51) for ub in (0, 1)
          for lb, Ms in (("lb1", (64, 1000)), ("lb1_d", (64, 1000)), ("lb2", (16,))) for M in Ms
          if not (lb == "lb1_d" and ub == 1)]


@pytest.mark.parametrize("inst,lb,ub,M", PARITY)
def test_rounds_match_reference_pool_loop(tmp_path, inst, lb, ub, M):
    step1, snaps, improved = oracle_search(inst, LB[lb], ub, 5, M, 1)
    got1, got = stop_after_one_call(tmp_path / "ck", inst, lb, ub, 5, M)
    assert got1 == step1
    compare(got, snaps[0])
    if ub == 0:  # leaves were reached and lowered the incumbent inside a chunk: the slow path ran and matched
        assert improved > 0 and got["best"] < 2**62


@pytest.mark.parametrize("inst,lb,ub", [(31, "lb1_d", 0), (41, "lb1", 1)])
def test_tiny_arena_compaction_and_growth(tmp_path, monkeypatch, inst, lb, ub):
    monkeypatch.setenv("TSB200_POOL_CAP", "3000")
    step1, snaps, _ = oracle_search(inst, LB[lb], ub, 5, 1000, 1)
    got1, got = stop_after_one_call(tmp_path / "ck", inst, lb, ub, 5, 1000)
    assert got1 == step1
    compare(got, snaps[0])


def test_resume_equals_uninterrupted_prefix(tmp_path):
    calls = 3
    step1, snaps, _ = oracle_search(31, LB["lb1"], 0, 5, 64, calls)
    path = tmp_path / "ck"
    for k in range(calls):
        got1, got = stop_after_one_call(path, 31, "lb1", 0, 5, 64)
        assert got1 == step1
        compare(got, snaps[k])


def test_checkpoint_widths_are_not_interchangeable(tmp_path):
    """a 50-job checkpoint is refused by the 20-job resumable search and the other way round, file untouched"""
    p50, p20 = tmp_path / "c50", tmp_path / "c20"
    stop_after_one_call(p50, 31, "lb1", 0, 5, 64)
    with pytest.raises(tsb200.SearchStopped):
        tsb200.pfsp_search_device(14, "lb1", 0, 5, 64, 1, checkpoint=str(p20), time_limit=0.0)
    b50, b20 = p50.read_bytes(), p20.read_bytes()
    L, st = tsb200.lib(), tsb200.SearchStats()
    assert L.tsb_pfsp_search_device_ckpt(31, 1, 0, 5, 64, 1, 1, os.fsencode(str(p50)), 0.0, C.byref(st)) == -1
    assert L.tsb_pfsp_search_device_ckpt_wide(50, 14, 1, 0, 5, 64, 1, 1, os.fsencode(str(p20)), 0.0, C.byref(st)) == -1
    assert p50.read_bytes() == b50 and p20.read_bytes() == b20

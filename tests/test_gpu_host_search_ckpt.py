"""The resumable host-pool searches (tsb_nq_search_ckpt, tsb_pfsp_search_ckpt, tsb_pfsp_search_ckpt_wide) on a GPU.

- Chains: the same call rerun until it returns TSB_OK, every invocation stopping after one offload per task
  (seconds = 0), ends with the stats of the uninterrupted twin in every field but the times and kernel_launches, for
  D = 1 and 2 and for ub 0 and 1 (host tasks never steal), and removes its file.
- A 50-job search that does not finish (ta031 lb1 ub 0): after k invocations its checkpoint's pool (in order),
  counters and incumbent are those of the oracle's pool loop after k chunks; the 50-job goldens pass through the
  resumable form too.
- A stop requested from another thread, and the Python interface's SearchStopped."""
import ctypes as C
import json
import os
import struct
import threading
import time
from collections import deque

import numpy as np
import pytest

import tsb200
from tsb200 import _lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "counts.json")))
GOLDEN50 = json.load(open(os.path.join(ROOT, "tests", "golden", "pfsp50_searches.json")))["searches"]
EXACT = ("explored_tree", "explored_sol", "best", "offloads", "offloaded_parents", "steals")
LB = {"lb1_d": 0, "lb1": 1, "lb2": 2}
M_TA002 = 100


@pytest.fixture(scope="module")
def L():
    return tsb200.lib()


def nq_call(L, path, N, M, D=1, max_queens=20, seconds=0.0):
    st = _lib.SearchStats()
    rc = L.tsb_nq_search_ckpt(max_queens, N, 1, 25, M, D, os.fsencode(str(path)), seconds, C.byref(st))
    return rc, st


def pfsp_call(L, path, inst, lb, ub, M, D=1, m=25, seconds=0.0):
    st = _lib.SearchStats()
    p = os.fsencode(str(path))
    if inst > 30:
        rc = L.tsb_pfsp_search_ckpt_wide(50, inst, lb, ub, m, M, D, p, seconds, C.byref(st))
    else:
        rc = L.tsb_pfsp_search_ckpt(inst, lb, ub, m, M, D, p, seconds, C.byref(st))
    return rc, st


def chain(call, path):
    """rerun `call` until the search ends: (final stats, invocations, the partial trees of the stops); each stop leaves
    a checkpoint at `path`, the end removes it"""
    n, trees = 0, []
    while True:
        rc, st = call()
        n += 1
        if rc != _lib.ESTOPPED:
            assert rc == _lib.OK, tsb200.lib().tsb_strerror(rc)
            assert not os.path.exists(path) and not os.path.exists(f"{path}.tmp")
            return st, n, trees
        assert os.path.getsize(path) > 0
        trees.append(st.explored_tree)
        assert n < 1000


def same(a, b, D):
    for f in EXACT:
        assert getattr(a, f) == getattr(b, f), f
    assert list(a.per_gpu_tree)[:D] == list(b.per_gpu_tree)[:D]
    # (a search that ends in step 1 launches nothing: ta037 lb1_d with D = 2)
    assert a.t_step2 > 0 and (a.kernel_launches > 0) == (a.offloads > 0)


def check_chain(got, n, trees, want, D):
    same(got, want, D)
    # every invocation but the last makes at least one offload and stops; the last one makes none (D = 1: exactly
    # one offload per stop)
    assert n >= 4
    if D == 1:
        assert n == want.offloads + 1
    assert trees == sorted(trees) and all(t <= got.explored_tree for t in trees)


# ------------------------------------------------------------------------------------------ chains
@pytest.mark.parametrize("D,M", [(1, 200000), (2, 200000)])
def test_nq13_chain_is_the_uninterrupted_search(L, tmp_path, D, M):
    path = tmp_path / "nq.ck"
    got, n, trees = chain(lambda: nq_call(L, path, 13, M, D), path)
    want = tsb200.nqueens_search(13, 1, 25, M, D)
    check_chain(got, n, trees, want, D)
    assert (got.explored_tree, got.explored_sol) == (GOLDEN["nqueens"]["13"]["tree"], GOLDEN["nqueens"]["13"]["sol"])


def test_nq12_wide_chain_is_the_uninterrupted_search(L, tmp_path):
    path = tmp_path / "nq24.ck"
    got, n, trees = chain(lambda: nq_call(L, path, 12, 40000, max_queens=24), path)
    want = tsb200.nqueens_search(12, 1, 25, 40000, 1, max_queens=24)
    check_chain(got, n, trees, want, 1)
    assert (got.explored_tree, got.explored_sol) == (GOLDEN["nqueens"]["12"]["tree"], GOLDEN["nqueens"]["12"]["sol"])


def test_pfsp_ta014_lb1_ub1_chain(L, tmp_path):
    path = tmp_path / "pf.ck"
    got, n, trees = chain(lambda: pfsp_call(L, path, 14, 1, 1, 100000), path)
    want = tsb200.pfsp_search(14, "lb1", 1, 25, 100000, 1)
    check_chain(got, n, trees, want, 1)
    g = GOLDEN["pfsp"]["ta014_lb1_ub1"]
    assert (got.explored_tree, got.explored_sol, got.best) == (g["tree"], g["sol"], g["best"])


def test_pfsp_ta002_lb2_ub0_two_tasks_chain(L, tmp_path):
    """ub = 0 with D = 2: each task prunes with its own incumbent; the device-pool form reproduces this only without
    stealing, the host-pool form always.  The search makes about 3 800 offloads at any M, so after three stops at one
    offload per task the chain stops every 0.2 s, wherever that falls"""
    path = tmp_path / "pf2.ck"
    calls = []

    def call():
        calls.append(0)
        return pfsp_call(L, path, 2, 2, 0, M_TA002, D=2, seconds=0.0 if len(calls) <= 3 else 0.2)

    got, n, trees = chain(call, path)
    want = tsb200.pfsp_search(2, "lb2", 0, 25, M_TA002, 2)
    check_chain(got, n, trees, want, 2)
    assert got.best == 1359 and got.offloads > 1000


@pytest.mark.parametrize("key", sorted(GOLDEN50))
def test_pfsp50_goldens_through_the_resumable_form(L, tmp_path, key):
    """m = 1: the root itself is offloaded, so every golden search makes at least one offload"""
    inst, lb = int(key[2:5]), key[6:]
    g = GOLDEN50[key]
    for D in (1, 2):
        path = tmp_path / f"{key}_{D}.ck"
        got, n, _ = chain(lambda: pfsp_call(L, path, inst, LB[lb], 1, 50000, D=D, m=1), path)
        want = tsb200.pfsp_search_wide(inst, lb, 1, 1, 50000, D)
        same(got, want, D)
        assert (got.explored_tree, got.explored_sol, got.best) == (g["tree"], g["sol"], g["best"]), (D, n)


# ------------------------------------------------------------------------------------------ ta031 against the oracle
def oracle_chunks(inst, lb, ub, m, M, chunks):
    """the oracle's pool loop (or_pfsp_expand_chunk: evaluate + the sequential generate_children): step 1 and the
    state after each of the first `chunks` chunks of popBackBulk(m, M)"""
    from oracle import pyoracle50 as po50
    Lo = po50.lib()
    Lo.or_pfsp_expand_chunk.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int64), C.c_void_p,
                                        C.c_int64, C.POINTER(C.c_uint64)]
    Lo.or_pfsp_expand_chunk.restype = C.c_int64
    t = po50.tables(inst)

    def expand(parents, best):
        parents = np.ascontiguousarray(parents)
        out = np.zeros(max(1, len(parents) * 50), dtype=po50.PFSP_NODE_DTYPE)
        b, sol = C.c_int64(best), C.c_uint64(0)
        k = Lo.or_pfsp_expand_chunk(C.byref(t), lb, parents.ctypes.data, len(parents), C.byref(b), out.ctypes.data,
                                    len(out), C.byref(sol))
        assert k >= 0
        return out[:k], int(sol.value), int(b.value)

    best = int(tsb200.lib().tsb_taillard_best_ub(inst)) if ub else 2**63 - 1
    root = np.zeros(1, dtype=po50.PFSP_NODE_DTYPE)
    root["limit1"] = -1
    root["prmu"][0] = np.arange(50)
    tree1 = sol1 = 0
    q = deque([root[0]])
    while len(q) < m and q:
        kids, s, best = expand(np.array([q.popleft()], dtype=po50.PFSP_NODE_DTYPE), best)
        tree1 += len(kids)
        sol1 += s
        q.extend(kids)
    buf = np.array(list(q), dtype=po50.PFSP_NODE_DTYPE)  # the pool is buf[:size], a stack
    size = len(buf)
    tree = sol = parents = 0
    snaps = []
    for k in range(chunks):
        assert size >= m
        n = min(size, M)
        size -= n
        kids, s, best = expand(buf[size:size + n], best)
        if size + len(kids) > len(buf):
            buf = np.concatenate([buf[:size], np.zeros(max(len(buf), len(kids)), dtype=buf.dtype)])
        buf[size:size + len(kids)] = kids
        size += len(kids)
        tree += len(kids)
        sol += s
        parents += n
        snaps.append(dict(tree=tree, sol=sol, offloads=k + 1, parents=parents, best=best, pool=buf[:size].tobytes()))
    return (tree1, sol1), snaps


def read_host_ckpt(path, rec=208):
    """the fields of a one-task host-pool checkpoint (layout: csrc/search_ckpt.cpp)"""
    b = open(path, "rb").read()
    assert b[:8] == b"TSB200CK"
    version, problem, r = struct.unpack_from("<3I", b, 8)
    assert (version, problem, r) == (1, 2, rec)
    assert struct.unpack_from("<7i", b, 20)[-1] == 0  # pools = 0: a host-pool search
    o = 20 + 7 * 4
    tree1, sol1, best1 = struct.unpack_from("<QQq", b, o)
    o += 24 + 16 + 8
    tree, sol, offloads, parents, launches, best, finished, pools, left = struct.unpack_from("<5Qq2IQ", b, o)
    o += 5 * 8 + 8 + 8 + 8
    assert finished == 0 and pools == 1 and left == 0
    pbest, count = struct.unpack_from("<qQ", b, o)
    o += 16
    assert pbest == best and len(b) == o + count * rec + 8
    return (tree1, sol1), dict(tree=tree, sol=sol, offloads=offloads, parents=parents, best=pbest,
                               pool=b[o:o + count * rec])


def test_ta031_lb1_ub0_stops_match_the_oracle_pool_loop(L, tmp_path):
    """a search that does not finish: after each of 64 invocations (one chunk each) the checkpoint is the oracle's pool
    loop after as many chunks.  M = 64, m = 5: every chunk takes the deepest nodes, so the first leaves (depth 50) come
    after about 49 chunks, and under ub = 0 they lower the incumbent inside a chunk"""
    m, M, calls = 5, 64, 64
    (tree1, sol1), snaps = oracle_chunks(31, LB["lb1"], 0, m, M, calls)
    path = tmp_path / "ck"
    for k in range(calls):
        rc, st = pfsp_call(L, path, 31, LB["lb1"], 0, M, m=m)
        assert rc == _lib.ESTOPPED
        got1, got = read_host_ckpt(path)
        assert got1 == (tree1, sol1)
        want = snaps[k]
        assert {f: got[f] for f in ("tree", "sol", "offloads", "parents", "best")} == \
            {f: want[f] for f in ("tree", "sol", "offloads", "parents", "best")}
        assert got["pool"] == want["pool"], f"pools differ ({len(got['pool']) // 208} vs {len(want['pool']) // 208})"
        assert st.explored_tree == tree1 + got["tree"] and st.offloads == k + 1
    assert snaps[-1]["best"] < 2**62  # (leaves were reached: the incumbent fell inside the chunks)


# ------------------------------------------------------------------------------------------ stop request, Python
def test_stop_request_from_another_thread(L, tmp_path):
    path = tmp_path / "n16.ck"
    asked = []

    def ask():
        time.sleep(0.5)
        asked.append(time.perf_counter())
        tsb200.request_stop()

    th = threading.Thread(target=ask)
    th.start()
    rc, st = nq_call(L, path, 16, 50000, seconds=-1)
    back = time.perf_counter()
    th.join()
    assert rc == _lib.ESTOPPED and path.exists()
    latency = back - asked[0]
    print(f"\nhost-pool N = 16 stop request to return: {latency * 1e3:.1f} ms; checkpoint {os.path.getsize(path)} bytes")
    assert 0 <= latency < 10
    assert 0 < st.explored_tree < GOLDEN["nqueens"]["16"]["tree"]
    rc, st = nq_call(L, path, 16, 50000, seconds=-1)  # (the request was cleared by the search that stopped on it)
    assert rc == _lib.OK and not path.exists()
    assert (st.explored_tree, st.explored_sol) == (GOLDEN["nqueens"]["16"]["tree"], GOLDEN["nqueens"]["16"]["sol"])


@pytest.mark.parametrize("search,args,golden", [
    (tsb200.nqueens_search, (12, 1, 25, 40000, 1), (856188, 14200, 0)),
    (tsb200.pfsp_search, (14, "lb1", 1, 25, 200000, 1), (2573652, 2648, 1377)),
    (tsb200.pfsp_search_wide, (37, "lb1", 1, 1, 50000, 1), (11, 0, 2725))])
def test_python_search_stopped(tmp_path, search, args, golden):
    path = tmp_path / "py.ck"
    partial = []
    while True:
        try:
            st = search(*args, checkpoint=path, time_limit=0)
            break
        except tsb200.SearchStopped as e:
            assert e.code == _lib.ESTOPPED and path.exists()
            partial.append(e.stats.explored_tree)
        assert len(partial) < 1000
    assert partial and not path.exists()
    assert (st.explored_tree, st.explored_sol, st.best) == golden
    assert all(0 <= t <= st.explored_tree for t in partial) and partial == sorted(partial)
    # without a time limit it runs to the end in one call
    st = search(*args, checkpoint=path)
    assert (st.explored_tree, st.explored_sol, st.best) == golden and not path.exists()

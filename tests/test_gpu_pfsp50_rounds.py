"""The persistent kernel of 50-job device pools (csrc/pfsp_wide_rounds.cuh, lb1 and lb1_d), through the resumable
device-pool search of a MAX_JOBS = 50 build (ta031..ta060) stopped after its first library call:

- route parity: the same search under TSB200_NO_ROUNDS=1 (the step loop of two-kernel rounds) leaves the same
  checkpoint, every field but the times and kernel_launches, on 5, 10 and 20 machines, one to four pools per task, with
  small chunks (M = 1, 64, 1 000), and with full chunks on both sides of the one-pool capacity and of the two-pool
  cutoff (the route switches inside the test): there m = M and a call is cut to two rounds (TSB200_CKPT_ROUNDS), so
  every round takes exactly M parents, full 384-parent slices on every SM, and the checkpoint stays small;
- each pool against the reference's pool loop (the oracle built with OR_MAX_JOBS = 50), with ub = 0, so that leaves
  lower the incumbent inside a chunk: the kernel's IMPROVED exit and the slow path that redoes that round are covered;
- PAUSE exactness (stops and resumes equal the uninterrupted pool loop), arena growth (SPACE) with a tiny arena, whole
  searches against the reference's goldens (trees of 0 to 11 nodes: a check of the search's plumbing, not of the
  kernel's paths), and that the kernel route costs a few launches per call, not two per round."""
import json
import os
import struct

import numpy as np
import pytest

import tsb200
from oracle import pyoracle50 as po50
from test_gpu_pfsp50_search import LB, REC, ROUNDS_PER_CALL, expand, golden, root

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "pfsp50_searches.json")))["searches"]
m = 5


def capacity(K):
    """parents per pool one launch of the kernel takes with K pools (csrc/pfr_tiers.h: 384 per CTA, one CTA per SM for
    one pool, two per SM shared by K pools, at most 256 per pool)"""
    sms = tsb200.lib().tsb_device_sm_count(0)
    return min(sms if K == 1 else 2 * sms // K, 256) * 384


def read_ckpt(path, K):
    """step 1, the task's counters and each pool (incumbent, nodes) of a one-task checkpoint (csrc/search_ckpt.cpp)"""
    b = open(path, "rb").read()
    assert b[:8] == b"TSB200CK"
    assert struct.unpack_from("<3I", b, 8) == (1, 2, REC)
    step1 = struct.unpack_from("<QQq", b, 48)
    tree, sol, offloads, parents, launches, best, finished, pools, left = struct.unpack_from("<5Qq2IQ", b, 96)
    assert finished == 0 and pools == K and left == 0
    o, out = 160, []
    for _ in range(K):
        pbest, count = struct.unpack_from("<qQ", b, o)
        out.append((pbest, b[o + 16:o + 16 + count * REC]))
        o += 16 + count * REC
    return step1, dict(tree=tree, sol=sol, offloads=offloads, parents=parents, best=best, pools=out), launches


def search(path, inst, lb, ub, M, K, m=m):
    """one library call of the resumable search (D = 1, K pools): ("stopped", checkpoint, launches) or, for a search
    that ends inside it, ("finished", counts, launches)"""
    if os.path.exists(path):
        os.remove(path)
    try:
        st = tsb200.pfsp_search_device_wide(inst, lb, ub, m, M, 1, K, checkpoint=str(path), time_limit=0.0)
    except tsb200.SearchStopped:
        step1, got, launches = read_ckpt(path, K)
        return "stopped", (step1, got), launches
    return "finished", (st.explored_tree, st.explored_sol, st.best, st.offloads, st.offloaded_parents), st.kernel_launches


def oracle_pools(inst, lb, ub, M, K, calls, m=m, rounds_per_call=ROUNDS_PER_CALL):
    """step 1 until the pool holds m K nodes, the search's strided split into K pools, and each pool's loop of
    popBackBulk(m, M) + expand for `calls` blocks of ROUNDS_PER_CALL rounds with its own incumbent; the state after
    each block, and how many rounds lowered an incumbent inside the chunk"""
    t = po50.tables(inst)
    best = int(tsb200.lib().tsb_taillard_best_ub(inst)) if ub else 2**63 - 1
    tree1 = sol1 = 0
    q, h = [root()[0]], 0
    while len(q) - h < m * K and h < len(q):
        kids, s, best = expand(t, lb, np.array([q[h]], dtype=po50.PFSP_NODE_DTYPE), best)
        h += 1
        tree1 += len(kids)
        sol1 += s
        q.extend(kids)
    q = q[h:]
    c = len(q) // K
    parts = [[q[g + i * K] for i in range(c)] + (q[K * c:] if g == K - 1 else []) for g in range(K)]
    pools = [dict(buf=np.array(p, dtype=po50.PFSP_NODE_DTYPE), best=best) for p in parts]
    tree = sol = offloads = parents = improved = 0
    snaps = []
    for _ in range(calls):
        for p in pools:
            buf, size = p["buf"], len(p["buf"])
            for _ in range(rounds_per_call):
                if size < m:
                    break
                n = min(size, M)
                size -= n
                kids, s, nb = expand(t, lb, buf[size:size + n], p["best"])
                improved += nb < p["best"]
                p["best"] = nb
                if size + len(kids) > len(buf):
                    buf = np.concatenate([buf[:size], np.zeros(max(len(buf), len(kids)), dtype=buf.dtype)])
                buf[size:size + len(kids)] = kids
                size += len(kids)
                tree += len(kids)
                sol += s
                offloads += 1
                parents += n
            p["buf"] = buf[:size]
        snaps.append(dict(tree=tree, sol=sol, offloads=offloads, parents=parents, best=min(p["best"] for p in pools),
                          pools=[(p["best"], p["buf"].tobytes()) for p in pools]))
    return (tree1, sol1, best), snaps, improved


def compare(got, want):
    assert {k: got[k] for k in ("tree", "sol", "offloads", "parents", "best")} == \
        {k: want[k] for k in ("tree", "sol", "offloads", "parents", "best")}
    for i, ((gb, gp), (wb, wp)) in enumerate(zip(got["pools"], want["pools"])):
        assert gb == wb, f"pool {i}: incumbent {gb} vs {wb}"
        assert gp == wp, f"pool {i} differs ({len(gp) // REC} vs {len(wp) // REC} nodes)"


# ------------------------------------------------------------------------------------------ 1. kernel against step loop
INSTANCES = (31, 41, 51)  # 5, 10 and 20 machines
SMALL_M = (1, 64, 1000)


# (lb1_d under ub = 1 prunes every child of the root of ta031 / ta041 / ta051: no round would run)
WORKLOADS = [("lb1", 0), ("lb1", 1), ("lb1_d", 0)]


def parity_cases():
    """(M = 1 000 under ub = 0 is test 2's, against the reference itself)"""
    for K in (1, 2, 3, 4):
        for inst in INSTANCES:
            for lb, ub in WORKLOADS:
                for M in SMALL_M[:2] if ub == 0 else SMALL_M:
                    yield K, inst, lb, ub, M


@pytest.mark.parametrize("K,inst,lb,ub,M", list(parity_cases()))
def test_kernel_matches_step_loop(tmp_path, monkeypatch, K, inst, lb, ub, M):
    monkeypatch.setenv("TSB200_NO_ROUNDS", "1")
    want = search(tmp_path / "a", inst, lb, ub, M, K)
    monkeypatch.delenv("TSB200_NO_ROUNDS")
    got = search(tmp_path / "b", inst, lb, ub, M, K)
    assert got[:2] == want[:2]
    if ub == 0 or lb == "lb1":  # (these run rounds: the comparison is not of two empty searches)
        assert got[1][1]["offloads"] > 0 if got[0] == "stopped" else got[1][3] > 0


FULL_ROUNDS = 2  # rounds per call in the full-chunk cases: the second reads what the first stored


def full_chunk_cases():
    """one pool at the one-pool capacity -1 / +0 / +1 (kernel, kernel, step loop); two pools at the shared cutoff
    (20 000: one shared launch; 20 001: the pools in turn, each in the one-pool kernel) and at the one-pool capacity
    (50 688: in turn; 50 689: step loop); three pools (in turn) at the three-pool capacity"""
    # (lb1_d under ub = 1 does have a tree on ta042 (10 machines) and ta054 (20); ub = 0 would grow pools of GBs here)
    for lb, ub, insts in (("lb1", 1, INSTANCES), ("lb1_d", 1, (42, 54))):
        for inst in insts:
            for K, M in ((1, ("cap", -1)), (1, ("cap", 0)), (1, ("cap", 1)), (2, 20000), (2, 20001),
                         (2, ("cap", 0)), (2, ("cap", 1)), (3, ("cap", 0))):
                if inst in (31, 54) and (K, M) not in ((1, ("cap", 0)), (2, 20000)):
                    continue  # (their pools grow 10 to 20 children per parent: GBs of checkpoint at these M)
                yield K, inst, lb, ub, M


def full_chunk_search(path, inst, lb, ub, M, K):
    kind, (step1, got), launches = search(path, inst, lb, ub, M, K, m=M)
    assert kind == "stopped"
    # every round of every pool took exactly M parents
    assert got["offloads"] == FULL_ROUNDS * K and got["parents"] == got["offloads"] * M, got["offloads"]
    return step1, got


@pytest.mark.parametrize("K,inst,lb,ub,M", list(full_chunk_cases()))
def test_full_chunks_kernel_matches_step_loop(tmp_path, monkeypatch, K, inst, lb, ub, M):
    if isinstance(M, tuple):
        M = capacity(K) + M[1]
    monkeypatch.setenv("TSB200_NO_STEAL", "1")
    monkeypatch.setenv("TSB200_CKPT_ROUNDS", str(FULL_ROUNDS))
    monkeypatch.setenv("TSB200_NO_ROUNDS", "1")
    want = full_chunk_search(tmp_path / "a", inst, lb, ub, M, K)
    monkeypatch.delenv("TSB200_NO_ROUNDS")
    got = full_chunk_search(tmp_path / "b", inst, lb, ub, M, K)
    assert got[0] == want[0]
    compare(got[1], want[1])


@pytest.mark.parametrize("K,inst,lb,ub,M", [(1, 41, "lb1", 1, 50688), (2, 31, "lb1", 1, 20000),
                                            (1, 54, "lb1_d", 1, 50688), (2, 51, "lb1", 1, 20000)])
def test_full_chunks_match_reference_pool_loop(tmp_path, monkeypatch, K, inst, lb, ub, M):
    monkeypatch.setenv("TSB200_NO_STEAL", "1")
    monkeypatch.setenv("TSB200_CKPT_ROUNDS", str(FULL_ROUNDS))
    step1, snaps, _ = oracle_pools(inst, LB[lb], ub, M, K, 1, m=M, rounds_per_call=FULL_ROUNDS)
    got1, got = full_chunk_search(tmp_path / "ck", inst, lb, ub, M, K)
    assert got1 == step1
    compare(got, snaps[0])


# ------------------------------------------------------------------------------------- 2. against the reference's loop
@pytest.mark.parametrize("K", [1, 2, 3, 4])
@pytest.mark.parametrize("inst", INSTANCES)
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
@pytest.mark.parametrize("M", [64, 1000])
def test_pools_match_reference_pool_loop(tmp_path, K, inst, lb, M):
    step1, snaps, improved = oracle_pools(inst, LB[lb], 0, M, K, 1)
    kind, (got1, got), _ = search(tmp_path / "ck", inst, lb, 0, M, K)
    assert kind == "stopped" and got1 == step1
    compare(got, snaps[0])
    assert improved > 0  # leaves lowered an incumbent inside a chunk: IMPROVED exits, rounds redone on the slow path


# ---------------------------------------------------------------------------------------------------- 3. PAUSE exactness
def test_resume_equals_uninterrupted_prefix_two_pools(tmp_path):
    calls = 3
    step1, snaps, _ = oracle_pools(31, LB["lb1"], 0, 64, 2, calls)
    path = tmp_path / "ck"
    for k in range(calls):
        with pytest.raises(tsb200.SearchStopped):
            tsb200.pfsp_search_device_wide(31, "lb1", 0, m, 64, 1, 2, checkpoint=str(path), time_limit=0.0)
        got1, got, _ = read_ckpt(path, 2)
        assert got1 == step1
        compare(got, snaps[k])


# -------------------------------------------------------------------------------------------------------- 4. SPACE
@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("inst,lb", [(31, "lb1_d"), (51, "lb1")])
def test_arena_grows_mid_call(tmp_path, monkeypatch, K, inst, lb):
    monkeypatch.setenv("TSB200_POOL_CAP", "3000")
    step1, snaps, _ = oracle_pools(inst, LB[lb], 0, 1000, K, 1)
    kind, (got1, got), _ = search(tmp_path / "ck", inst, lb, 0, 1000, K)
    assert kind == "stopped" and got1 == step1
    compare(got, snaps[0])


# ------------------------------------------------------------------------------------------------- 5. whole searches
@pytest.mark.parametrize("m_", [1, 25])
@pytest.mark.parametrize("key", sorted(k for k in GOLDEN if not k.endswith("lb2")))
def test_whole_searches_match_reference(key, m_):
    inst, lb = int(key[2:5]), key[6:]
    for D in (1, 2):
        for pools in (1, 2, 3, 4):
            M = min(20000, capacity(pools))  # (every K takes the kernel)
            st = tsb200.pfsp_search_device_wide(inst, lb, 1, m_, M, D, pools)
            assert (st.explored_tree, st.explored_sol, st.best) == golden(key), (D, pools, st.explored_tree)


# ------------------------------------------------------------------------------------------------ 6. the route is taken
@pytest.mark.parametrize("K", [1, 2, 4])
def test_kernel_route_takes_few_launches(tmp_path, monkeypatch, K):
    monkeypatch.setenv("TSB200_NO_STEAL", "1")  # (1024 rounds of every pool in the call)
    kind, (_, got), launches = search(tmp_path / "a", 31, "lb1", 1, 1000, K)
    assert kind == "stopped" and got["offloads"] >= 100 * K
    # (two pools share each launch; four take the one-pool kernel in turn: a few launches per pool)
    assert launches <= (8 if K <= 2 else 8 * K), (launches, got["offloads"])
    # (the search counts the launches of its first pool's handle: two per round of that pool on the step loop)
    monkeypatch.setenv("TSB200_NO_ROUNDS", "1")
    _, (_, want), step_launches = search(tmp_path / "b", 31, "lb1", 1, 1000, K)
    assert want["offloads"] == got["offloads"] and step_launches >= 200

"""PFSP device-pool searches with several device pools per task (tsb_pfsp_search_device_pools, _part, and
tsb_pfsp_search_on_pools): pools = 1 is the one-pool search field for field; with K pools per task every pool is one
reference task, so D = 1 is the reference's run with D = K tasks (po.pfsp_search_offload) and D > 1 is a two-level
split of the warm-up pool, checked against an emulation below built from the oracle's chunk step (po.pfsp_expand).

ub = 0 is checked on lb2 only: a search with lb1 / lb1_d from an infinite incumbent is far too large for the oracle
(minutes for one run).  ta002 (20 jobs x 5 machines) keeps the lb2 ub = 0 oracle runs to a few seconds each."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po

M_SMALL = 25
EINVAL = tsb200._lib.EINVAL
PFR_SLICE, PFR_MAX_CTAS = 384, 256  # csrc/pfr_tiers.h
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200", "drivers", "pfsp_b200.out")


def pool_capacity(sms, pools):
    """pfr_tiers.h pf_pool_capacity (tests/test_pfr_tiers.py checks the formula against the header)"""
    return min(sms if pools <= 1 else 2 * sms // pools, PFR_MAX_CTAS) * PFR_SLICE


@pytest.fixture
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


@pytest.fixture(autouse=True)
def default_env(monkeypatch):
    """no switch of the library leaks in from the caller's environment"""
    for v in ("TSB200_NO_STEAL", "TSB200_NO_ROUNDS", "TSB200_POOLS", "TSB200_NO_SIMD16", "TSB200_POOL_CAP"):
        monkeypatch.delenv(v, raising=False)


@pytest.fixture
def sms(gpu):
    n = int(tsb200.lib().tsb_device_sm_count(0))
    assert n > 0
    return n


def golden(name):
    return json.load(open(os.path.join(ROOT, "tests", "golden", name)))


def totals(st):
    return (st.explored_tree, st.explored_sol, st.best, st.offloads, st.offloaded_parents)


def fields(st):
    """every field of tsb_search_stats except the times"""
    return totals(st) + (st.kernel_launches, tuple(st.per_gpu_tree), st.steals)


def oracle_totals(r):
    return (r.tree, r.sol, r.best, r.offloads, r.offloaded_parents)


def call(fn, *args):
    st = tsb200.SearchStats()
    rc = fn(*args, C.byref(st))
    return rc, st


# ------------------------------------------------------------------------------------------ pools = 1
@pytest.mark.gpu
@pytest.mark.parametrize("inst,lb,ub,M,D", [(14, "lb1", 1, 50000, 1), (14, "lb2", 0, 3000, 2)])
def test_one_pool_is_the_one_pool_search(inst, lb, ub, M, D, gpu):
    L, kind = tsb200.lib(), tsb200.LB_NAMES[lb]
    rc0, old = call(L.tsb_pfsp_search_device, inst, kind, ub, M_SMALL, M, D)
    rc1, new = call(L.tsb_pfsp_search_device_pools, inst, kind, ub, M_SMALL, M, D, 1)
    assert rc0 == rc1 == 0 and fields(new) == fields(old)
    for part in range(D):
        rc0, old = call(L.tsb_pfsp_search_device_part, inst, kind, ub, M_SMALL, M, D, part, 0)
        rc1, new = call(L.tsb_pfsp_search_device_pools_part, inst, kind, ub, M_SMALL, M, D, 1, part, 0)
        assert rc0 == rc1 == 0 and fields(new) == fields(old), part


# ------------------------------------------------------------------------------------------ D = 1: the reference
def m_values(sms, K):
    return {"300": 300, "6000": 6000, "cap": pool_capacity(sms, K), "cap+1": pool_capacity(sms, K) + 1}


CASES_UB1 = [(14, lb, K, Mk) for lb in ("lb1", "lb1_d") for K in (2, 3, 4) for Mk in ("300", "6000", "cap", "cap+1")]
CASES_UB1 += [(14, "lb2", K, Mk) for K in (2, 3, 4) for Mk in ("300", "6000")] + [(20, "lb2", 2, "6000")]


@pytest.mark.gpu
@pytest.mark.parametrize("inst,lb,K,Mk", CASES_UB1)
def test_one_task_is_the_reference_with_K_tasks(inst, lb, K, Mk, sms, monkeypatch):
    """ub = 1 and D = 1: K pools = the reference's run with K tasks (same warm-up, split, chunks); in one launch per
    call of the persistent kernel for lb1 / lb1_d within the K-pool capacity, one pool after the other beyond it"""
    M = m_values(sms, K)[Mk]
    want = po.pfsp_search_offload(inst, tsb200.LB_NAMES[lb], 1, M_SMALL, M, K)
    monkeypatch.setenv("TSB200_NO_STEAL", "1")
    st = tsb200.pfsp_search_device(inst, lb, 1, M_SMALL, M, 1, pools=K)
    assert totals(st) == oracle_totals(want)
    assert st.per_gpu_tree[0] == sum(want.task_tree[:K]) and st.steals == 0
    with tsb200.PfspEvaluator(inst, M=M) as ev:
        one_launch = ev.pools_per_launch(lb, M) >= K
    assert one_launch == (lb != "lb2" and M <= pool_capacity(sms, K))
    if one_launch:
        assert 0 < st.kernel_launches < max(24, st.offloads // 4 + 24)
    # with moves between the pools: the chunks change, what the whole search explores does not
    monkeypatch.delenv("TSB200_NO_STEAL")
    st = tsb200.pfsp_search_device(inst, lb, 1, M_SMALL, M, 1, pools=K)
    assert totals(st)[:3] == oracle_totals(want)[:3]


@pytest.mark.gpu
@pytest.mark.parametrize("K,M", [(2, 300), (3, 300), (4, 300), (2, 6000)])
def test_falling_incumbents_on_one_handle(K, M, gpu):
    """ub = 0, lb2 on a handle the caller owns (tsb_pfsp_search_on_pools): K incumbents that leaves lower mid-search
    (rounds redone by the sequential rule), the reference's K-task counts, twice on the same handles"""
    inst = 2
    want = po.pfsp_search_offload(inst, tsb200.LB2, 0, M_SMALL, M, K)
    with tsb200.PfspEvaluator(inst, M=M) as ev:
        evs = [ev] + [ev.sibling(i) for i in range(1, K)]
        for _ in range(2):
            slow = [e.slow_rounds for e in evs]
            st = ev.search(inst, "lb2", 0, M_SMALL, M, pools=K)
            assert totals(st) == oracle_totals(want)
            assert st.per_gpu_tree[0] == sum(want.task_tree[:K]) and st.steals == 0
            assert sum(e.slow_rounds - s for e, s in zip(evs, slow)) > 0
            assert all(e.pool_size == 0 for e in evs)


# ------------------------------------------------------------------------------------------ D > 1
def root_node(jobs):
    r = np.zeros(1, dtype=po.PFSP_NODE_DTYPE)
    r["limit1"] = -1
    r["prmu"][0, :jobs] = np.arange(jobs)
    return r


def strided_split(nodes, D):
    """static_split of the reference's multi-GPU drivers: node g + i D to part g, the remainder to the last part"""
    n = nodes.shape[0]
    c = n // D
    parts = [nodes[g:g + c * D:D] for g in range(D)]
    parts[-1] = np.concatenate([parts[-1], nodes[D * c:]])
    return parts


def run_pool(t, kind, nodes, best, m, M):
    """the oracle's chunk loop on one pool: popBackBulk(m, M), evaluate + generate_children"""
    pool, tree, sol, offloads, parents = nodes, 0, 0, 0, 0
    while pool.shape[0] >= m:
        n = min(pool.shape[0], M)
        chunk, pool = np.ascontiguousarray(pool[-n:]), pool[:-n]
        kids, s, best = po.pfsp_expand(t, kind, chunk, best)
        tree, sol, offloads, parents = tree + kids.shape[0], sol + s, offloads + 1, parents + n
        pool = np.concatenate([pool, kids])
    return pool, tree, sol, best, offloads, parents


def emulate_two_level(inst, kind, m, M, D, K):
    """step 1 to D K m nodes, the strided split into D shares and of every share into K pools, each pool's chunk loop
    with its own incumbent, the leftovers handed back pool by pool (popBack), min-reduce, step 3 (popBack +
    decompose, one parent per expand)"""
    t = po.tables(inst)
    best = 2**63 - 1
    pool = root_node(t.jobs)
    tree = sol = 0
    while pool.shape[0] < D * K * m:  # step 1: popFront + decompose
        kids, s, best = po.pfsp_expand(t, kind, np.ascontiguousarray(pool[:1]), best)
        pool = np.concatenate([pool[1:], kids])
        tree, sol = tree + kids.shape[0], sol + s
    offloads = parents = 0
    per_task, bests, rest = [], [best], []
    for share in strided_split(pool, D):
        task_tree = 0
        for nodes in strided_split(share, K):
            left, tr, s, b, o, p = run_pool(t, kind, nodes, best, m, M)
            task_tree, sol, offloads, parents = task_tree + tr, sol + s, offloads + o, parents + p
            bests.append(b)
            rest.append(left[::-1])
        per_task.append(task_tree)
        tree += task_tree
    best = min(bests)
    rest = np.concatenate(rest)
    while rest.shape[0]:  # step 3
        parent, rest = rest[-1:].copy(), rest[:-1]
        kids, s, best = po.pfsp_expand(t, kind, parent, best)
        rest = np.concatenate([rest, kids])
        tree, sol = tree + kids.shape[0], sol + s
    return (tree, sol, best, offloads, parents), per_task


@pytest.mark.gpu
@pytest.mark.parametrize("D", [2, 3])
def test_tasks_with_falling_incumbents_are_the_two_level_split(D, gpu):
    """ub = 0, K = 2: nothing moves between pools or tasks; the counts are the emulation's (tasks wrap onto however
    many GPUs exist)"""
    K, M = 2, 300
    want, per_task = emulate_two_level(2, tsb200.LB2, M_SMALL, M, D, K)
    st = tsb200.pfsp_search_device(2, "lb2", 0, M_SMALL, M, D, pools=K)
    assert totals(st) == want and st.steals == 0
    assert list(st.per_gpu_tree[:D]) == per_task and all(x == 0 for x in st.per_gpu_tree[D:])


@pytest.mark.gpu
@pytest.mark.parametrize("D", [2, 3])
@pytest.mark.parametrize("lb,M", [("lb1", 3000), ("lb1", 50000), ("lb2", 3000)])
def test_tasks_with_stealing_keep_the_reference_totals(lb, M, D, gpu):
    want = golden("counts.json")["pfsp"][f"ta014_lb{tsb200.LB_NAMES[lb]}_ub1"]
    st = tsb200.pfsp_search_device(14, lb, 1, M_SMALL, M, D, pools=2)
    assert (st.explored_tree, st.explored_sol, st.best) == (want["tree"], want["sol"], want["best"])
    assert sum(st.per_gpu_tree[:D]) <= st.explored_tree and all(x == 0 for x in st.per_gpu_tree[D:])


@pytest.mark.gpu
@pytest.mark.parametrize("D", [2, 3])
def test_parts_add_up_to_the_whole_search(D, gpu):
    """ub = 1: the parts (one process per GPU) add up to the whole search and to the reference's counts"""
    want = golden("counts.json")["pfsp"]["ta014_lb1_ub1"]
    whole = tsb200.pfsp_search_device(14, "lb1", 1, M_SMALL, 3000, D, pools=2)
    got = [tsb200.pfsp_search_device_part(14, "lb1", 1, M_SMALL, 3000, D, p, pools=2) for p in range(D)]
    for p, st in enumerate(got):
        assert sum(st.per_gpu_tree) == st.per_gpu_tree[p] and st.steals == 0 and st.best == want["best"], p
    assert (sum(st.explored_tree for st in got), sum(st.explored_sol for st in got)) == (want["tree"], want["sol"])
    assert (whole.explored_tree, whole.explored_sol) == (want["tree"], want["sol"])


# ------------------------------------------------------------------------------------------ arguments (no GPU)
@pytest.mark.parametrize("pools", [0, 5, -1])
def test_pool_count_is_checked(pools):
    L = tsb200.lib()
    assert call(L.tsb_pfsp_search_device_pools, 14, 1, 1, M_SMALL, 1000, 1, pools)[0] == EINVAL
    assert call(L.tsb_pfsp_search_device_pools_part, 14, 1, 1, M_SMALL, 1000, 2, pools, 0, 0)[0] == EINVAL
    with pytest.raises(tsb200.TsbError) as ex:
        tsb200.pfsp_search_device(14, "lb1", 1, M_SMALL, 1000, 1, pools=pools)
    assert ex.value.code == EINVAL


def test_null_arguments_are_refused():
    L = tsb200.lib()
    assert L.tsb_pfsp_search_device_pools(14, 1, 1, M_SMALL, 1000, 1, 2, None) == EINVAL
    assert L.tsb_pfsp_search_device_pools_part(14, 1, 1, M_SMALL, 1000, 2, 2, 0, 0, None) == EINVAL
    assert call(L.tsb_pfsp_search_on_pools, None, 14, 1, 1, M_SMALL, 1000, 2)[0] == EINVAL


@pytest.mark.parametrize("args", [(31, 1, 1, M_SMALL, 1000, 1), (0, 1, 1, M_SMALL, 1000, 1),
                                  (14, 3, 1, M_SMALL, 1000, 1), (14, 1, 2, M_SMALL, 1000, 1),
                                  (14, 1, 1, 0, 1000, 1), (14, 1, 1, M_SMALL, 0, 1), (14, 1, 1, M_SMALL, 1000, 9)])
def test_refusals_are_the_one_pool_search_refusals(args):
    """an instance (a 50-job one, none), bound, ub, m, M or D the one-pool search refuses: the same code"""
    L = tsb200.lib()
    want = call(L.tsb_pfsp_search_device, *args)[0]
    assert want != 0
    assert call(L.tsb_pfsp_search_device_pools, *args, 2)[0] == want
    assert call(L.tsb_pfsp_search_device_pools_part, *args, 2, 0, 0)[0] == want


# ------------------------------------------------------------------------------------------ driver
def run_driver(*args):
    assert os.path.exists(DRIVER), f"{DRIVER} is missing: build() makes it"
    return subprocess.run([DRIVER, *map(str, args)], capture_output=True, text=True, timeout=600)


@pytest.mark.parametrize("args", [("--pools", 2), ("--pools", 0), ("--pools", 5, "--devpool", 1)])
def test_driver_pool_arguments(args):
    r = run_driver(*args)
    assert r.returncode == 2 and "--pools" in r.stderr and "Size of the explored tree" not in r.stdout


def test_driver_help_names_pools():
    r = run_driver("--help")
    assert r.returncode == 1 and "--pools" in r.stdout


@pytest.mark.gpu
def test_driver_two_pools_is_the_reference_with_two_tasks(gpu, monkeypatch):
    monkeypatch.setenv("TSB200_NO_STEAL", "1")
    want = po.pfsp_search_offload(14, tsb200.LB1, 1, M_SMALL, 50000, 2)
    r = run_driver("--inst", 14, "--lb", "lb1", "--ub", 1, "--devpool", 1, "--pools", 2)
    assert r.returncode == 0, r.stderr
    got = [int(re.search(p, r.stdout).group(1)) for p in
           (r"Size of the explored tree: (\d+)", r"Number of explored solutions: (\d+)", r"Optimal makespan: (\d+)",
            r"offloads: (\d+)")]
    assert got == [want.tree, want.sol, want.best, want.offloads]

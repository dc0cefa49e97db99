"""Whole PFSP searches whose counts depend on how the incumbent moves (lb2 with ub = 0, per-task incumbents of the
D-way split) and the process-per-GPU parts of the N-Queens and PFSP searches, against the oracle's offload search
(tests/golden/pfsp_searches.json, tests/golden/make_golden_searches.py) and its part search."""
import json
import os

import pytest

import tsb200
from oracle import pyoracle as po
from test_gpu_nq_boards import pool_capacity

pytestmark = pytest.mark.gpu

M_SMALL = 25


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


def pinned():
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pfsp_searches.json")
    return json.load(open(here))["searches"]


SEARCHES = pinned()


def totals(st):
    return (st.explored_tree, st.explored_sol, st.best, st.offloads, st.offloaded_parents)


def want_totals(e):
    return (e["tree"], e["sol"], e["best"], e["offloads"], e["offloaded_parents"])


@pytest.fixture
def default_env(monkeypatch):
    monkeypatch.delenv("TSB200_NO_STEAL", raising=False)
    monkeypatch.delenv("TSB200_POOLS", raising=False)


# ------------------------------------------------------------------------------------------ whole searches
@pytest.mark.parametrize("mode", ["host", "device"])
@pytest.mark.parametrize("key", list(SEARCHES))
def test_pinned_search(key, mode, default_env, monkeypatch):
    """host pool (tsb_pfsp_search) and device pool (tsb_pfsp_search_device) against the oracle; with ub = 0 the
    library must not steal (the counts would depend on timing), so every task's step 2 is the oracle task's"""
    e = SEARCHES[key]
    D = e["D"]
    run = tsb200.pfsp_search if mode == "host" else tsb200.pfsp_search_device
    steals = mode == "device" and e["ub"] == 1 and D > 1  # the one case in which the device pools steal
    if steals:  # the static split alone first: the oracle's chunk sequence, task by task
        monkeypatch.setenv("TSB200_NO_STEAL", "1")
    st = run(e["inst"], e["lb"], e["ub"], M_SMALL, e["M"], D)
    assert st.steals == 0
    assert totals(st) == want_totals(e)
    assert list(st.per_gpu_tree[:D]) == e["task_tree"] and all(x == 0 for x in st.per_gpu_tree[D:])
    if steals:
        # with stealing, a steal moves nodes between tasks and changes the chunks, and so which nodes are left for
        # step 3: only what the whole search explores stays the same
        monkeypatch.delenv("TSB200_NO_STEAL")
        st = run(e["inst"], e["lb"], e["ub"], M_SMALL, e["M"], D)
        assert totals(st)[:3] == want_totals(e)[:3]
        assert sum(st.per_gpu_tree[:D]) < st.explored_tree and all(x == 0 for x in st.per_gpu_tree[D:])


@pytest.mark.parametrize("key", [k for k, e in SEARCHES.items() if e["lb"] == "lb2" and e["ub"] == 0 and e["D"] == 1])
def test_lb2_falling_incumbent_on_one_handle(key):
    """the D = 1 lb2 searches on a handle the caller owns, twice: rounds in which a leaf lowers best are redone by
    the sequential rule (slow rounds), and nothing of the first search (incumbent, round bookkeeping) leaks into
    the second"""
    e = SEARCHES[key]
    with tsb200.PfspEvaluator(e["inst"], M=e["M"]) as ev:
        st = ev.search(e["inst"], "lb2", 0, M_SMALL, e["M"])
        assert totals(st) == want_totals(e) and st.per_gpu_tree[0] == e["task_tree"][0]
        slow = ev.slow_rounds
        assert slow > 0
        st = ev.search(e["inst"], "lb2", 0, M_SMALL, e["M"])
        assert totals(st) == want_totals(e) and st.per_gpu_tree[0] == e["task_tree"][0]
        assert ev.slow_rounds > slow


# ------------------------------------------------------------------------------------------ PFSP parts
PART_KEYS = [k for k, e in SEARCHES.items() if "parts" in e]


@pytest.mark.parametrize("key", PART_KEYS)
def test_pfsp_parts(key, golden_dir, default_env):
    """every part of the split against the oracle's part; with ub = 1 the parts add up to the whole search and to
    the reference's count"""
    e = SEARCHES[key]
    D = e["D"]
    got = [tsb200.pfsp_search_device_part(e["inst"], e["lb"], e["ub"], M_SMALL, e["M"], D, p) for p in range(D)]
    for p, (st, w) in enumerate(zip(got, e["parts"])):
        assert totals(st) == want_totals(w), p
        assert st.per_gpu_tree[p] == w["task_tree"][p] == e["task_tree"][p]
        assert sum(st.per_gpu_tree) == st.per_gpu_tree[p] and st.steals == 0
    assert e["ub"] == 1
    assert (sum(st.explored_tree for st in got), sum(st.explored_sol for st in got)) == (e["tree"], e["sol"])
    ref = json.load(open(os.path.join(golden_dir, "counts.json")))["pfsp"][f"ta{e['inst']:03d}_lb{tsb200.LB_NAMES[e['lb']]}_ub1"]
    assert (e["tree"], e["sol"], e["best"]) == (ref["tree"], ref["sol"], ref["best"])


@pytest.mark.parametrize("key", [k for k, e in SEARCHES.items() if e["ub"] == 0 and e["D"] > 1])
def test_pfsp_parts_with_their_own_incumbents(key, default_env):
    """ub = 0: a part's step 2 is that task's step 2 in the whole search (same start, same best from step 1); its
    step 3 then prunes with the best it found itself, and the best of all parts is the optimum"""
    e = SEARCHES[key]
    D = e["D"]
    got = [tsb200.pfsp_search_device_part(e["inst"], e["lb"], 0, M_SMALL, e["M"], D, p) for p in range(D)]
    for p, st in enumerate(got):
        assert st.per_gpu_tree[p] == e["task_tree"][p], p
        assert st.best <= e["task_best"][p] and st.steals == 0
    assert min(st.best for st in got) == e["best"]


# ------------------------------------------------------------------------------------------ N-Queens parts
def pools_wanted(sms, M, cap=4):
    """nq_pools_wanted: the most pools (up to cap) whose persistent-kernel capacity takes chunks of M"""
    for P in range(cap, 1, -1):
        if M <= pool_capacity(sms, P):
            return P
    return 1


@pytest.mark.parametrize("N", [12, 13])
@pytest.mark.parametrize("D", [2, 3, 5])
@pytest.mark.parametrize("pools", ["1", None])
def test_nq_parts(N, D, pools, golden_dir, monkeypatch):
    monkeypatch.delenv("TSB200_NO_STEAL", raising=False)
    if pools is None:
        monkeypatch.delenv("TSB200_POOLS", raising=False)
    else:
        monkeypatch.setenv("TSB200_POOLS", pools)
    M = 50000
    sms = int(tsb200.lib().tsb_device_sm_count(0))
    P = 1 if pools == "1" else pools_wanted(sms, M)
    warm = D * M_SMALL * P
    got = [tsb200.nqueens_search_device_part(N, 1, M_SMALL, M, D, p) for p in range(D)]
    for p, st in enumerate(got):
        w = po.nq_search_offload_part(N, 1, M_SMALL, M, D, p, warm)
        assert (st.explored_tree, st.explored_sol) == (w.tree, w.sol), p
        assert st.steals == 0 and sum(st.per_gpu_tree) == st.per_gpu_tree[p]
        if P == 1:  # one pool per part: the reference's chunk sequence
            assert (st.offloads, st.offloaded_parents, st.per_gpu_tree[p]) == (w.offloads, w.offloaded_parents,
                                                                            w.task_tree[p])
    c = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    assert (sum(st.explored_tree for st in got), sum(st.explored_sol for st in got)) == (c["tree"], c["sol"])


# ------------------------------------------------------------------------------------------ arguments
@pytest.mark.parametrize("D,part", [(2, -1), (2, 2), (3, 5), (9, 0), (9, 8)])
def test_part_arguments(D, part):
    for call in (lambda: tsb200.nqueens_search_device_part(10, 1, M_SMALL, 1000, D, part),
                 lambda: tsb200.pfsp_search_device_part(14, "lb1", 1, M_SMALL, 1000, D, part)):
        with pytest.raises(tsb200.TsbError) as ex:
            call()
        assert ex.value.code == tsb200._lib.EINVAL

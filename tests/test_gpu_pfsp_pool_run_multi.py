"""Several independent PFSP device pools in one launch of the persistent kernel (tsb_pfsp_pool_run_multi,
csrc/pfsp_rounds.cuh) against the oracle's pool loop, pool by pool: each pool must end exactly where
tsb_pfsp_pool_run alone would leave it, so each is compared with its own OraclePfspPool (counters, incumbent, size,
drained bytes and slow_rounds after every call).  Covered: the capacity edges of 2, 3 and 4 pools and the fallback
one past them, ragged pools that leave the launch at different rounds, runs resumed over several calls, per-pool
incumbents with an IMPROVED exit in one pool only, a SPACE exit in one pool, one launch for all pools, instances
mixed in one launch, lb2, the argument checks, and the ta014 tree split over four pools to exhaustion.

Every size that depends on the GPU is derived at run time from tsb_device_sm_count with the formulas of
csrc/pfr_tiers.h (ctas_per_pool, pool_capacity below; tests/test_pfr_tiers.py checks them against the header)."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po
from test_gpu_pfsp_rounds import (INT64_MAX, JOBS, NODE, OPT, PF_TILE, PFR_MAX_CTAS, PFR_SLICE, OraclePfspPool,
                                  assert_pool, improved, live_bounds, median_bound, nodes, roots)

pytestmark = pytest.mark.gpu

PFR_MAX_POOLS = 4
EINVAL, EUNSUPPORTED = tsb200._lib.EINVAL, tsb200._lib.EUNSUPPORTED
EXIT_SPACE, EXIT_IMPROVED = 2, 5  # nq_rounds_ll.cuh RND_EXIT_SPACE, pfsp_rounds.cuh PFR_EXIT_IMPROVED


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


@pytest.fixture(autouse=True)
def default_routes(monkeypatch):
    """no environment switch of the library leaks in from the caller's environment"""
    for v in ("TSB200_NO_SIMD16", "TSB200_NO_ROUNDS", "TSB200_POOL_CAP", "TSB200_ROUNDS_PROF"):
        monkeypatch.delenv(v, raising=False)


@pytest.fixture(scope="module")
def sms():
    n = int(tsb200.lib().tsb_device_sm_count(0))
    assert n > 0
    return n


# ------------------------------------------------------------------------------------------ pfr_tiers.h
def ctas_per_pool(sms, pools):
    """pfr_tiers.h pf_ctas_per_pool: one pool: one CTA per SM; several: two CTAs per SM in all"""
    most = sms if pools <= 1 else 2 * sms // pools
    return min(most, PFR_MAX_CTAS)


def pool_capacity(sms, pools):
    """pfr_tiers.h pf_pool_capacity: the largest chunk of each pool"""
    return ctas_per_pool(sms, pools) * PFR_SLICE


# ------------------------------------------------------------------------------------------ helpers
def pools_of(ev, K):
    """ev and its first K - 1 siblings"""
    return [ev] + [ev.sibling(i) for i in range(1, K)]


def run_multi_and_check(evs, os_, lb, m, M, bests, max_rounds):
    """one pool_run_multi call against each pool's oracle loop: counters, incumbent, size and slow_rounds of every
    pool; -> the incumbents after the call"""
    slow0 = [ev.slow_rounds for ev in evs]
    r0 = [len(o.rounds) for o in os_]
    got = tsb200.pfsp_pool_run_multi(evs, lb, m, M, bests, max_rounds=max_rounds)
    after = []
    for i, (ev, o) in enumerate(zip(evs, os_)):
        want, wbest = o.run(m, M, bests[i], max_rounds)
        assert list(got[i][:4]) == want and got[i][4] == wbest, (i, M, max_rounds, got[i], want, wbest)
        assert ev.pool_size == o.size, i
        assert ev.slow_rounds - slow0[i] == sum(improved(r) for r in o.rounds[r0[i]:]), i
        after.append(wbest)
    return after


def run_multi_calls(evs, os_, lb, m, M, bests, calls):
    for k in calls:
        bests = run_multi_and_check(evs, os_, lb, m, M, bests, k)
    return bests


def assert_pools(evs, os_, push_back=True):
    for ev, o in zip(evs, os_):
        assert_pool(ev, o, push_back)


def push_all(evs, starts, t, lb):
    os_ = []
    for ev, s in zip(evs, starts):
        if s.shape[0]:
            ev.pool_push(s)
        os_.append(OraclePfspPool(t, lb, s))
    return os_


def prof_exits(text):
    """(pool, pools in the launch, rounds, exit code) of every launch, from the TSB200_ROUNDS_PROF lines"""
    return [tuple(int(x) for x in g) for g in
            re.findall(r"PFSP rounds kernel \(pool (\d+) of (\d+)\): (\d+) rounds \(exit (\d+)\)", text)]


# ------------------------------------------------------------------------------------------ capacity edges
@pytest.mark.parametrize("scalar", [False, True], ids=["simd16", "scalar"])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
@pytest.mark.parametrize("inst", [14, 21])
def test_capacity_edges(inst, lb, scalar, sms, monkeypatch):
    """K = 2, 3, 4 pools at M = 1, 128 G - 1, 128 G, 128 G + 1 (G = CTAs per pool), the K-pool capacity (one launch
    for the first round of every pool) and the capacity + 1 (the pools run one after the other)"""
    if scalar:
        monkeypatch.setenv("TSB200_NO_SIMD16", "1")
    t = po.tables(inst, heads_mode=0)
    rng = np.random.default_rng(9900 + 10 * inst + 2 * (lb == "lb1") + scalar)
    best = median_bound(t, lb, rng, 4, 14)
    M_max = pool_capacity(sms, 2) + 1
    with tsb200.PfspEvaluator(inst, M=M_max) as ev:
        if scalar:
            assert not ev.route & tsb200.ROUTE_SIMD16
        for K in (2, 3, 4):
            evs = pools_of(ev, K)
            assert len({x.route for x in evs}) == 1
            G, cap = ctas_per_pool(sms, K), pool_capacity(sms, K)
            assert ev.pools_per_launch(lb, cap) >= K and ev.pools_per_launch(lb, cap + 1) < K
            for M in sorted({1, PF_TILE * G - 1, PF_TILE * G, PF_TILE * G + 1, cap, cap + 1}):
                # pool 0 holds more than M (a full chunk), the others 2 G + 1 (every sub-slice of their CTAs
                # non-empty) or M // 2 + 1 (kept small: the oracle's rounds are what this test spends its time on)
                sizes = [M + 37] + [min(M, 2 * G + 1)] * (K - 2) + [min(M // 2 + 1, 3000)]
                starts = [nodes(rng, n, 4, 14) for n in sizes]
                os_ = push_all(evs, starts, t, lb)
                launches = ev.kernel_launches
                bests = run_multi_and_check(evs, os_, lb, 1, M, [best] * K, 1)
                assert os_[0].rounds[0]["parents"] == M
                if M <= cap:  # every pool's first round in one launch
                    assert ev.kernel_launches == launches + 1, (K, M)
                assert_pools(evs, os_)
                run_multi_calls(evs, os_, lb, 1 if M < 25 else 25, M, bests, (1,))
                assert_pools(evs, os_, push_back=False)


# ------------------------------------------------------------------------------------------ ragged pools, resuming
@pytest.mark.parametrize("M", [300, 6000])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_ragged_pools(lb, M):
    """four pools of very different sizes: one empty, one below m, one of deep nodes that is DONE after a round or
    two, one that goes on for many rounds; in calls of 1, 2, 3 and 40 rounds, each resuming from the stack the
    last launch left"""
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9910 + M + (lb == "lb1"))
    starts = [np.zeros(0, dtype=NODE), nodes(rng, 20, 4, 10), nodes(rng, 60, 18, 19), nodes(rng, 3 * M, 3, 9)]
    with tsb200.PfspEvaluator(14, M=M) as ev:
        evs = pools_of(ev, 4)
        os_ = push_all(evs, starts, t, lb)
        run_multi_calls(evs, os_, lb, 25, M, [OPT[14]] * 4, (1, 2, 3, 40))
        assert_pools(evs, os_, push_back=False)
    n = [len(o.rounds) for o in os_]
    assert n[0] == 0 and n[1] == 0 and 1 <= n[2] <= 3 and n[3] > n[2] + 3, n


@pytest.mark.parametrize("K", [2, 3, 4])
def test_resume_over_many_calls(K):
    """the same pools in calls of 1, 1, 2, 5 and 9 rounds against one call of 18: identical pools"""
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9920 + K)
    starts = [nodes(rng, 200 * (i + 1), 3, 12) for i in range(K)]
    with tsb200.PfspEvaluator(14, M=300) as a, tsb200.PfspEvaluator(14, M=300) as b:
        ea, eb = pools_of(a, K), pools_of(b, K)
        oa, ob = push_all(ea, starts, t, "lb1_d"), push_all(eb, starts, t, "lb1_d")
        run_multi_calls(ea, oa, "lb1_d", 25, 300, [OPT[14]] * K, (1, 1, 2, 5, 9))
        run_multi_calls(eb, ob, "lb1_d", 25, 300, [OPT[14]] * K, (18,))
        for x, y in zip(ea, eb):
            assert x.pool_drain().tobytes() == y.pool_drain().tobytes()


# ------------------------------------------------------------------------------------------ incumbents, SPACE
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_per_pool_incumbents(lb, capfd, monkeypatch):
    """three pools with the same chunk of depth-19 parents on top (smallest leaf bound L) and their own incumbents:
    best = L + 1 (pool 0: the first round leaves the kernel with IMPROVED and is redone by pool_step, best becomes
    L), best = L (pool 1: a tie, stays in the kernel) and best = L + 1 again on a pool whose chunk has no leaf (pool
    2).  Pools 1 and 2 keep running in the launch pool 0 left: the call takes exactly the launches pool 0 alone takes"""
    monkeypatch.setenv("TSB200_ROUNDS_PROF", "1")
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9930 + (lb == "lb1"))
    below, chunk = nodes(rng, 300, 8, 12), nodes(rng, 500, 19, 19)
    b, _ = live_bounds(t, lb, chunk)
    L = int(b[:, 19].min())
    starts = [np.concatenate([below, chunk]), np.concatenate([below, chunk]), nodes(rng, 800, 8, 12)]
    bests = [L + 1, L, L + 1]
    with tsb200.PfspEvaluator(14, M=500) as single:
        single.pool_push(starts[0])
        single.pool_run(lb, 1, 500, L + 1, max_rounds=3)
        alone = single.kernel_launches
    capfd.readouterr()
    with tsb200.PfspEvaluator(14, M=500) as ev:
        evs = pools_of(ev, 3)
        os_ = push_all(evs, starts, t, lb)
        launches = ev.kernel_launches
        after = run_multi_and_check(evs, os_, lb, 1, 500, bests, 3)
        assert ev.kernel_launches - launches == alone
        assert after == [L, L, L + 1]
        assert [ev.slow_rounds for ev in evs] == [1, 0, 0]
        assert [len(o.rounds) for o in os_] == [3, 3, 3]
        assert_pools(evs, os_)
        run_multi_calls(evs, os_, lb, 1, 500, after, (2, 4))
        assert_pools(evs, os_, push_back=False)
    first = prof_exits(capfd.readouterr().err)[:3]
    assert first == [(0, 3, 0, EXIT_IMPROVED), (1, 3, 3, 1), (2, 3, 3, 1)], first


@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_space_exit_in_one_pool(lb, capfd, monkeypatch):
    """an arena of 1 080 records (TSB200_POOL_CAP) in every pool: pool 0 starts from 54 roots, whose second round
    does not fit (a SPACE exit; the arena grows and the pool goes again) while pools 1 and 2 (at most 25 nodes of
    depth 18 - 19, at most 2 children each) always fit"""
    monkeypatch.setenv("TSB200_POOL_CAP", str(JOBS * 54))
    monkeypatch.setenv("TSB200_ROUNDS_PROF", "1")
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9940 + (lb == "lb1"))
    starts = [roots(rng, 54), nodes(rng, 20, 18, 19), nodes(rng, 25, 18, 19)]
    with tsb200.PfspEvaluator(14, M=300) as ev:
        evs = pools_of(ev, 3)
        os_ = push_all(evs, starts, t, lb)
        capfd.readouterr()
        run_multi_calls(evs, os_, lb, 1, 300, [OPT[14]] * 3, (6, 6))
        assert_pools(evs, os_, push_back=False)
    exits = prof_exits(capfd.readouterr().err)
    # the first launch: pool 0 leaves for room after one round, pools 1 and 2 go on
    assert exits[0] == (0, 3, 1, EXIT_SPACE) and all(e[1] == 3 and e[3] != EXIT_SPACE for e in exits[1:3]), exits


# ------------------------------------------------------------------------------------------ one launch
@pytest.mark.parametrize("K", [2, 3, 4])
def test_one_launch_for_all_pools(K, sms):
    """no IMPROVED round, arenas large enough: K pools, 2 rounds each, one launch in all; at the K-pool capacity"""
    M = pool_capacity(sms, K)
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9950 + K)
    best = median_bound(t, "lb1", rng, 3, 12)
    starts = [nodes(rng, M + 100 * i, 3, 12) for i in range(K)]
    with tsb200.PfspEvaluator(14, M=M) as ev:
        evs = pools_of(ev, K)
        os_ = push_all(evs, starts, t, "lb1")
        launches = ev.kernel_launches
        run_multi_and_check(evs, os_, "lb1", 25, M, [best] * K, 2)
        assert ev.kernel_launches == launches + 1
        assert all(len(o.rounds) == 2 and not any(improved(r) for r in o.rounds) for o in os_)
        assert_pools(evs, os_, push_back=False)


# ------------------------------------------------------------------------------------------ instances, lb2
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_mixed_instances(lb):
    """ta014 and ta015 (same route, different tables) share a launch, each with its own tables and incumbent"""
    rng = np.random.default_rng(9960 + (lb == "lb1"))
    t14, t15 = po.tables(14, heads_mode=0), po.tables(15, heads_mode=0)
    b14, b15 = median_bound(t14, lb, rng, 4, 14), median_bound(t15, lb, rng, 4, 14)
    s = [nodes(rng, 700, 4, 14), nodes(rng, 500, 4, 14)]
    with tsb200.PfspEvaluator(14, M=300) as e14, tsb200.PfspEvaluator(15, M=300) as e15:
        assert e14.route == e15.route
        e14.pool_push(s[0])
        e15.pool_push(s[1])
        os_ = [OraclePfspPool(t14, lb, s[0]), OraclePfspPool(t15, lb, s[1])]
        launches = e14.kernel_launches + e15.kernel_launches
        bests = run_multi_and_check([e14, e15], os_, lb, 25, 300, [b14, b15], 1)
        assert e14.kernel_launches + e15.kernel_launches == launches + 1
        run_multi_calls([e14, e15], os_, lb, 25, 300, bests, (3, 50))
        assert_pools([e14, e15], os_, push_back=False)


def test_lb2_runs_the_pools_one_after_the_other():
    """lb2 has no persistent kernel: the pools run one after the other through pool_run, with the oracle's results"""
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9970)
    starts = [nodes(rng, 150 * (i + 1), 6, 16) for i in range(3)]
    with tsb200.PfspEvaluator(14, M=300) as ev:
        assert ev.pools_per_launch("lb2", 300) == 1 and ev.pools_per_launch("lb1", 300) == PFR_MAX_POOLS
        evs = pools_of(ev, 3)
        os_ = push_all(evs, starts, t, "lb2")
        run_multi_calls(evs, os_, "lb2", 25, 300, [OPT[14]] * 3, (1, 4))
        assert_pools(evs, os_, push_back=False)


# ------------------------------------------------------------------------------------------ arguments
def raw_multi(handles, n, lb=tsb200.LB1, M=300, bests=None):
    hs = (C.c_void_p * max(1, len(handles)))(*handles)
    b = (C.c_int64 * PFR_MAX_POOLS)(*([OPT[14]] * PFR_MAX_POOLS if bests is None else bests))
    out = (C.c_uint64 * (4 * 8))()
    return tsb200.lib().tsb_pfsp_pool_run_multi(hs, n, lb, 1, M, 10, b, out)


def test_arguments(monkeypatch):
    L = tsb200.lib()
    with tsb200.PfspEvaluator(14, M=300) as ev, tsb200.PfspEvaluator(14, M=300) as other:
        h = [ev._h.value] + [ev.sibling(i)._h.value for i in (1, 2, 3)]
        assert len(set(h)) == 4 and ev._h.value not in h[1:]
        assert raw_multi(h[:2], 2) == 0
        assert raw_multi(h, 0) == EINVAL
        assert raw_multi(h + [other._h.value], 5) == EINVAL
        assert raw_multi([h[0], None], 2) == EINVAL
        assert raw_multi([h[0], h[1], h[0]], 3) == EINVAL
        assert raw_multi(h[:2], 2, M=301) == EINVAL
        assert raw_multi(h[:2], 2, lb=3) == EINVAL
        assert L.tsb_pfsp_pool_run_multi(None, 1, 1, 1, 300, 10, None, None) == EINVAL
        # siblings: index 1..3, the same handle on every call
        s = C.c_void_p()
        assert L.tsb_pfsp_sibling(ev._h, 0, C.byref(s)) == EINVAL
        assert L.tsb_pfsp_sibling(ev._h, 4, C.byref(s)) == EINVAL
        assert L.tsb_pfsp_sibling(ev._h, 2, C.byref(s)) == 0 and s.value == h[2]
        assert L.tsb_pfsp_sibling(ev._h, 2, C.byref(s)) == 0 and s.value == h[2]
        assert ev.sibling(2) is ev.sibling(2) and ev.sibling(2).route == ev.route
        # a sibling's launches count in its owner's tally
        launches = ev.kernel_launches
        ev.sibling(3).pool_push(nodes(np.random.default_rng(1), 50, 4, 10))
        ev.sibling(3).pool_run("lb1", 1, 300, OPT[14], max_rounds=1)
        assert ev.kernel_launches == launches + 1 and ev.sibling(3).kernel_launches == 1
        # different routes: 20 machines, or the scalar route of the same instance
        with tsb200.PfspEvaluator(21, M=300) as e21:
            assert raw_multi([h[0], e21._h.value], 2) == EINVAL
        monkeypatch.setenv("TSB200_NO_SIMD16", "1")
        with tsb200.PfspEvaluator(14, M=300) as sc:
            assert sc.route != ev.route and raw_multi([h[0], sc._h.value], 2) == EINVAL
        monkeypatch.delenv("TSB200_NO_SIMD16")
        # a wide (50-job) handle
        with tsb200.PfspEvaluator(41, M=300) as w:
            assert raw_multi([w._h.value, h[0]], 2) == EUNSUPPORTED
            assert raw_multi([h[0], w._h.value], 2) == EUNSUPPORTED
            assert L.tsb_pfsp_sibling(w._h, 1, C.byref(s)) == EUNSUPPORTED
        with pytest.raises(ValueError):
            tsb200.pfsp_pool_run_multi([ev, other], "lb1", 1, 300, [OPT[14]])
    assert L.tsb_pfsp_pools_per_launch(None, 1, 300) == 1


# ------------------------------------------------------------------------------------------ exhaustion
def test_root_split_over_four_pools_to_exhaustion(golden_dir):
    """ta014 lb1 under ub = 1: the root's pushed children, split strided into 4 pools (the reference's static
    split), m = 1, to exhaustion: the root's children plus every pool's children are the tree of counts.json"""
    want = json.load(open(os.path.join(golden_dir, "counts.json")))["pfsp"]["ta014_lb1_ub1"]
    t = po.tables(14, heads_mode=0)
    root = roots(np.random.default_rng(0), 1)
    kids, sol0, best = po.pfsp_expand(t, tsb200.LB1, root.view(po.PFSP_NODE_DTYPE), OPT[14])
    kids = kids.view(NODE)
    assert best == OPT[14] and kids.shape[0] > PFR_MAX_POOLS
    M = 20000
    with tsb200.PfspEvaluator(14, M=M) as ev:
        evs = pools_of(ev, PFR_MAX_POOLS)
        for i, e in enumerate(evs):
            e.pool_push(np.ascontiguousarray(kids[i::PFR_MAX_POOLS]))
        got = tsb200.pfsp_pool_run_multi(evs, "lb1", 1, M, [OPT[14]] * PFR_MAX_POOLS)
        assert all(e.pool_size == 0 and e.slow_rounds == 0 for e in evs)
        assert all(g[4] == OPT[14] and g[0] > 0 for g in got)
    assert kids.shape[0] + sum(g[2] for g in got) == want["tree"]
    assert sol0 + sum(g[3] for g in got) == want["sol"]

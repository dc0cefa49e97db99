"""GPU tests of the fused evaluate + generate_children path and of the device-resident pool (SURVEY §8f rows 1, 3):
children arrays byte-identical to the oracle's generate_children output, pools byte-identical after the same
rounds, and whole searches with the reference's counts."""
import json
import os

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po
from test_gpu_parity import rand_nq

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("N", [1, 4, 8, 13, 17, 19, 20])
def test_expand_matches_oracle_children(N):
    rng = np.random.default_rng(500 + N)
    with tsb200.NQueensEvaluator(N, M=20000) as ev:
        for count, lo in ((1, 0), (3, 0), (511, 0), (512, 0), (513, 2), (4096 + 17, 0), (20000, max(0, N - 6))):
            parents = rand_nq(rng, N, count, depth_lo=min(lo, N))
            got, gsol = ev.expand(parents)
            want, wsol = po.nq_expand(parents.view(po.NQ_NODE_DTYPE), N)
            assert gsol == wsol and got.shape[0] == want.shape[0]
            assert got.tobytes() == want.tobytes()


def test_expand_dense_tiles_take_the_unstaged_path():
    """depth 0/1 parents have up to N children each: far more than a tile's staging image holds"""
    N = 17
    rng = np.random.default_rng(9)
    parents = rand_nq(rng, N, 3000, depth_lo=0, depth_hi=1)
    with tsb200.NQueensEvaluator(N, M=3000) as ev:
        got, gsol = ev.expand(parents)
    want, wsol = po.nq_expand(parents.view(po.NQ_NODE_DTYPE), N)
    assert gsol == wsol == 0 and got.tobytes() == want.tobytes() and got.shape[0] > 3000 * 10


@pytest.mark.parametrize("N,which", [(12, 3), (14, 100)])
def test_expand_on_captured_real_chunks(N, which):
    parents = po.nq_capture_chunk(N, which).view(tsb200.NQ_NODE_DTYPE)
    with tsb200.NQueensEvaluator(N, M=50000) as ev:
        got, gsol = ev.expand(parents)
    want, wsol = po.nq_expand(parents.view(po.NQ_NODE_DTYPE), N)
    assert gsol == wsol and got.tobytes() == want.tobytes()


def test_device_pool_is_byte_identical_to_the_reference_pool():
    """run the reference's offload loop (popBackBulk(m, M) -> evaluate -> generate_children -> pushBack) on the
    host with the oracle and on the device with tsb_nq_pool_*; the pools must agree after every round"""
    N, m, M = 11, 25, 700
    rng = np.random.default_rng(4)
    start = rand_nq(rng, N, 60, depth_lo=1, depth_hi=3)
    host = [start[i:i + 1] for i in range(start.shape[0])]
    host_pool = start.copy()
    with tsb200.NQueensEvaluator(N, M=M) as ev:
        ev.pool_push(start)
        for _ in range(40):
            n_par, n_child, n_sol = ev.pool_step(m, M)
            if host_pool.shape[0] < m:
                assert n_par == 0
                break
            n = min(host_pool.shape[0], M)
            chunk = np.ascontiguousarray(host_pool[host_pool.shape[0] - n:])
            kids, sol = po.nq_expand(chunk.view(po.NQ_NODE_DTYPE), N)
            host_pool = np.concatenate([host_pool[: host_pool.shape[0] - n], kids.view(tsb200.NQ_NODE_DTYPE)])
            assert (n_par, n_child, n_sol) == (n, kids.shape[0], sol)
            assert ev.pool_size == host_pool.shape[0]
        rest = ev.pool_drain()
        assert rest.tobytes() == np.ascontiguousarray(host_pool).tobytes() and ev.pool_size == 0
    del host


def test_device_pool_compaction_and_growth(golden_dir, monkeypatch):
    """a tiny arena (TSB200_POOL_CAP) forces the extent stack to be compacted into the second arena and the
    arenas to grow many times during a search; counts and chunk sequence must not change"""
    monkeypatch.setenv("TSB200_POOL_CAP", "3000")
    monkeypatch.setenv("TSB200_POOLS", "1")  # one pool per task: the reference's D = 1 chunk sequence
    N, m, M = 12, 25, 500
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    st = tsb200.nqueens_search_device(N, 1, m, M)
    ref = po.nq_search_offload(N, 1, m, M, 1)
    assert (st.explored_tree, st.explored_sol) == (counts["tree"], counts["sol"])
    assert (st.offloads, st.offloaded_parents) == (ref.offloads, ref.offloaded_parents)


@pytest.mark.parametrize("N,m,M,D", [(10, 25, 50000, 1), (12, 25, 50000, 1), (12, 5, 300, 1), (13, 25, 4096, 1),
                                     (14, 25, 50000, 1), (15, 25, 1 << 20, 1), (13, 25, 2000, 3), (14, 25, 50000, 4)])
def test_device_resident_search_counts(golden_dir, N, m, M, D, monkeypatch):
    monkeypatch.setenv("TSB200_NO_STEAL", "1")  # the static split alone: the reference driver's chunk sequence
    monkeypatch.setenv("TSB200_POOLS", "1")     # ... with one pool per task
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    st = tsb200.nqueens_search_device(N, 1, m, M, D)
    assert (st.explored_tree, st.explored_sol) == (counts["tree"], counts["sol"])
    ref = po.nq_search_offload(N, 1, m, M, D)  # same chunk sequence as the reference driver
    assert (st.offloads, st.offloaded_parents) == (ref.offloads, ref.offloaded_parents)
    if M <= 512 * 100:  # the persistent multi-round kernel: a handful of launches for all rounds
        assert 0 < st.kernel_launches < max(16, st.offloads // 4 + 16)
    else:
        assert st.kernel_launches == 2 * st.offloads  # count, build


@pytest.mark.parametrize("N,m,M,P", [(10, 25, 50000, 4), (12, 5, 300, 4), (13, 25, 4096, 2), (14, 25, 50000, 4),
                                     (15, 25, 50000, 2), (15, 25, 50000, 4), (14, 25, 60000, 4)])
def test_several_pools_per_task_is_the_reference_split_into_as_many_tasks(golden_dir, N, m, M, P, monkeypatch):
    """default for chunks that fit the persistent kernel: the task's pool is split once more (the reference's strided
    split) into P device pools whose rounds share one launch (tsb_nq_pool_run_multi; P = 4 for M <= 50688 on an H100,
    else as many as one launch of the persistent kernel takes).  Without stealing, D = 1 is then exactly the
    reference's D = P run: same warm-up, same split, same chunk sequence in each pool"""
    monkeypatch.setenv("TSB200_NO_STEAL", "1")
    monkeypatch.setenv("TSB200_POOLS", str(P))
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    st = tsb200.nqueens_search_device(N, 1, m, M, 1)
    assert (st.explored_tree, st.explored_sol) == (counts["tree"], counts["sol"])
    # the tiers of the persistent kernel, from the SM count: four pools of SMs / 2 CTAs x 768 parents, else three of
    # 2 SMs / 3 CTAs x 768 (only tiers of several pools occur in the cases above)
    sms = min(tsb200.lib().tsb_device_sm_count(0), 256)
    pools = min(P, 4 if M <= 768 * (sms // 2) else 3)
    assert M <= 768 * (2 * sms // 3)
    with tsb200.NQueensEvaluator(N, 1, M) as ev:
        assert min(P, ev.pools_per_launch(M)) == pools
    ref = po.nq_search_offload(N, 1, m, M, pools)
    assert (st.offloads, st.offloaded_parents) == (ref.offloads, ref.offloaded_parents)
    assert 0 < st.kernel_launches < max(24, st.offloads // 4 + 24)


@pytest.mark.parametrize("N,m,M,D", [(13, 25, 2000, 1), (15, 25, 50000, 1), (14, 25, 50000, 3), (15, 25, 30000, 8)])
def test_several_pools_per_task_with_stealing_totals(golden_dir, N, m, M, D, monkeypatch):
    monkeypatch.delenv("TSB200_POOLS", raising=False)
    monkeypatch.delenv("TSB200_NO_STEAL", raising=False)
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    st = tsb200.nqueens_search_device(N, 1, m, M, D)
    assert (st.explored_tree, st.explored_sol) == (counts["tree"], counts["sol"])


@pytest.mark.parametrize("N,m,M,K", [(12, 25, 700, 2), (14, 25, 50000, 2), (13, 5, 3000, 3), (11, 25, 700, 4), (15, 25, 1 << 17, 2)])
def test_pool_run_multi_equals_separate_pool_runs(N, m, M, K):
    """K pools in shared launches of the persistent kernel against each pool run on its own: same counters, byte-
    identical leftovers (K > 2 or chunks beyond the persistent kernel: served one after the other by the library)"""
    rng = np.random.default_rng(N * 77 + K)
    starts = [rand_nq(rng, N, 40 + 13 * i, depth_lo=1, depth_hi=2) for i in range(K)]
    multi = [tsb200.NQueensEvaluator(N, M=M) for _ in range(K)]
    try:
        for ev, st in zip(multi, starts):
            ev.pool_push(st)
        got = tsb200.nqueens_pool_run_multi(multi, m, M, 10 ** 9)
        for i, st in enumerate(starts):
            with tsb200.NQueensEvaluator(N, M=M) as one:
                one.pool_push(st)
                want = one.pool_run(m, M, 10 ** 9)
                assert got[i] == want
                assert multi[i].pool_size == one.pool_size
                assert multi[i].pool_drain().tobytes() == one.pool_drain().tobytes()
        # a bounded number of rounds per pool
        for ev, st in zip(multi, starts):
            ev.pool_push(st)
        part = tsb200.nqueens_pool_run_multi(multi, m, M, 3)
        assert all(x[0] <= 3 for x in part)
        rest = tsb200.nqueens_pool_run_multi(multi, m, M, 10 ** 9)
        assert [tuple(a + b for a, b in zip(x, y)) for x, y in zip(part, rest)] == got
    finally:
        for ev in multi:
            ev.close()


@pytest.mark.parametrize("N,m,M,D", [(13, 25, 2000, 3), (14, 25, 50000, 4), (15, 25, 50000, 8), (15, 25, 1 << 18, 4),
                                     (12, 5, 300, 2)])
def test_device_resident_search_with_work_stealing(golden_dir, N, m, M, D):
    """D tasks (wrapping onto the GPUs present), device pools, stealing between them: the totals are those of the
    reference whatever the steals did to the per-GPU shares"""
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    st = tsb200.nqueens_search_device(N, 1, m, M, D)
    assert (st.explored_tree, st.explored_sol) == (counts["tree"], counts["sol"])
    assert sum(st.per_gpu_tree[:D]) <= st.explored_tree


def test_pool_steal_moves_the_oldest_half_in_order():
    N, m = 12, 25
    rng = np.random.default_rng(12)
    nodes = rand_nq(rng, N, 1001, depth_lo=1, depth_hi=5)
    with tsb200.NQueensEvaluator(N, M=5000) as victim, tsb200.NQueensEvaluator(N, M=5000) as thief:
        victim.pool_push(nodes)
        own = rand_nq(rng, N, 7, depth_lo=1, depth_hi=5)
        thief.pool_push(own)
        assert thief.pool_steal_from(victim, m) == 500  # size / 2 from the front (Pool_par.chpl:178-191)
        assert (victim.pool_size, thief.pool_size) == (501, 507)
        assert thief.pool_steal_from(victim, 300) == 0 and victim.pool_size == 501  # below 2 m: nothing moves
        assert thief.pool_drain().tobytes() == np.concatenate([own, nodes[:500]]).tobytes()
        assert victim.pool_drain().tobytes() == np.ascontiguousarray(nodes[500:]).tobytes()
        # and the pools keep working after a steal: the stolen half explored by the thief, the rest by the victim
        victim.pool_push(nodes[:200])
        assert thief.pool_steal_from(victim, m) == 100
        a, b = victim.pool_run(1, 5000), thief.pool_run(1, 5000)
    with tsb200.NQueensEvaluator(N, M=5000) as one:
        one.pool_push(nodes[:200])
        c = one.pool_run(1, 5000)
    assert a[2] + b[2] == c[2] and a[3] + b[3] == c[3]


# (M = 67000: just below the largest chunk one pool's persistent kernel takes on an H100, 512 parents x 132 SMs)
@pytest.mark.parametrize("N,m,M,rounds", [(11, 25, 700, 40), (12, 5, 300, 200), (13, 25, 5000, 37), (14, 25, 50000, 11),
                                          (17, 25, 50000, 6), (10, 1, 67000, 50), (8, 25, 50000, 1000)])
def test_pool_run_equals_the_same_number_of_pool_steps(N, m, M, rounds):
    """tsb_nq_pool_run (persistent cooperative kernel, children stored in place) against tsb_nq_pool_step (two
    kernels per round, extent stack): same counters, byte-identical pool, round by round and in bulk; and against
    the oracle's sequential rule"""
    rng = np.random.default_rng(N * 1000 + M)
    start = rand_nq(rng, N, 60, depth_lo=1, depth_hi=2)
    with tsb200.NQueensEvaluator(N, M=M) as a, tsb200.NQueensEvaluator(N, M=M) as b:
        a.pool_push(start)
        b.pool_push(start)
        tot = [0, 0, 0, 0]
        done = 0
        for _ in range(rounds):
            n_par, n_child, n_sol = a.pool_step(m, M)
            if n_par == 0:
                break
            done += 1
            tot = [tot[0] + 1, tot[1] + n_par, tot[2] + n_child, tot[3] + n_sol]
        # the same rounds in three launches of the persistent kernel: 1 round, a few, the rest
        got = [0, 0, 0, 0]
        for k in (1, 3, rounds):
            r = b.pool_run(m, M, min(k, rounds - got[0]))
            got = [x + y for x, y in zip(got, r)]
        assert got == tot and a.pool_size == b.pool_size
        ra, rb = a.pool_drain(), b.pool_drain()
        assert ra.tobytes() == rb.tobytes()
        assert b.kernel_launches <= 5  # three launches of the rounds kernel (+ the fat-arena import / export)


def test_pool_run_against_the_oracle_rule_and_growth(monkeypatch):
    """a tiny arena (TSB200_POOL_CAP) makes the persistent kernel leave for more room several times"""
    monkeypatch.setenv("TSB200_POOL_CAP", "2000")
    N, m, M = 11, 25, 700
    rng = np.random.default_rng(44)
    start = rand_nq(rng, N, 60, depth_lo=1, depth_hi=3)
    host_pool = start.copy()
    tot = [0, 0, 0, 0]
    for _ in range(25):
        if host_pool.shape[0] < m:
            break
        n = min(host_pool.shape[0], M)
        chunk = np.ascontiguousarray(host_pool[host_pool.shape[0] - n:])
        kids, sol = po.nq_expand(chunk.view(po.NQ_NODE_DTYPE), N)
        host_pool = np.concatenate([host_pool[: host_pool.shape[0] - n], kids.view(tsb200.NQ_NODE_DTYPE)])
        tot = [tot[0] + 1, tot[1] + n, tot[2] + kids.shape[0], tot[3] + sol]
    with tsb200.NQueensEvaluator(N, M=M) as ev:
        ev.pool_push(start)
        assert list(ev.pool_run(m, M, 25)) == tot
        assert ev.pool_drain().tobytes() == np.ascontiguousarray(host_pool).tobytes()


def test_pool_run_to_exhaustion_counts(golden_dir):
    """the whole step 2 of N = 13 in one call, m = 1: the pool runs empty; children + 1 root = explored tree"""
    N = 13
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    root = np.zeros(1, dtype=tsb200.NQ_NODE_DTYPE)
    root["board"][0, :N] = np.arange(N)
    with tsb200.NQueensEvaluator(N, M=50000) as ev:
        ev.pool_push(root)
        nr, npar, nc, ns = ev.pool_run(1, 50000)
        assert (nc, ns) == (counts["tree"], counts["sol"]) and npar == nc + 1 and ev.pool_size == 0

"""The device-pool search driver's step 2 (tsb_nq_search_on) against the same loop written over the pool primitives,
as bench.py's `value` writes it: the warm-up pool of step 1, the strided split into P device pools, dry pools taking
the oldest half of the fullest one, shared launches of at most 2048 rounds per pool, then the drain.  Where the
driver calls the library decides where dry pools rebalance, and so the rounds, the parents, the children and the
launches of the search: these must be the emulation's, one for one."""
import numpy as np
import pytest

import tsb200
from test_gpu_nq_boards import pool_capacity

pytestmark = pytest.mark.gpu

N, m, M = 15, 25, 5000  # every one of 4 pools runs well over 2048 rounds
INT64_MAX = 2**63 - 1


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


def pools_wanted(cap):
    """the driver's pools per task before a handle exists: TSB200_POOLS capped by ll_tiers.h ll_pools_for"""
    sms = int(tsb200.lib().tsb_device_sm_count(0))
    tier = 4 if M <= pool_capacity(sms, 4) else 3 if M <= pool_capacity(sms, 3) else 2 if M <= pool_capacity(sms, 1) else 1
    return min(cap, tier)


def emulated_step2(P, wanted):
    """(rounds, parents, children, launches) of step 2 on P fresh handles, and the most rounds one pool ran"""
    evs = [tsb200.NQueensEvaluator(N, 1, M) for _ in range(P)]
    try:
        warm, _, _ = tsb200.nqueens_warmup(N, wanted * m)
        c = warm.shape[0] // P
        for g, e in enumerate(evs):  # static_split: strided, the remainder to the last part
            part = warm[g:P * c:P] if g < P - 1 else np.concatenate([warm[g:P * c:P], warm[P * c:]])
            e.pool_push(np.ascontiguousarray(part))
        per_pool = np.zeros((P, 4), dtype=np.int64)
        if P == 1:
            per_pool[0] += evs[0].pool_run(m, M, INT64_MAX)
        else:
            floor = 2 * m  # steal_floor for chunks the persistent kernel takes
            while True:
                sizes = [e.pool_size for e in evs]
                for i, e in enumerate(evs):
                    if sizes[i] < m:
                        v = max(range(P), key=lambda j: sizes[j])
                        if v != i and sizes[v] >= floor:
                            e.pool_steal_from(evs[v], m)
                            sizes = [x.pool_size for x in evs]
                if max(sizes) < m:
                    break
                per_pool += np.array(tsb200.nqueens_pool_run_multi(evs, m, M, 2048), dtype=np.int64)
        for e in evs:
            e.pool_drain()
        launches = sum(e.kernel_launches for e in evs)
    finally:
        for e in evs:
            e.close()
    rounds, parents, children, _ = per_pool.sum(axis=0)
    return (int(rounds), int(parents), int(children), int(launches)), int(per_pool[:, 0].max())


@pytest.mark.parametrize("pools", [None, "1"])
def test_search_on_is_the_pool_loop(pools, monkeypatch):
    monkeypatch.delenv("TSB200_NO_STEAL", raising=False)
    if pools is None:
        monkeypatch.delenv("TSB200_POOLS", raising=False)
    else:
        monkeypatch.setenv("TSB200_POOLS", pools)
    wanted = pools_wanted(4 if pools is None else int(pools))
    with tsb200.NQueensEvaluator(N, 1, M) as ev:
        P = min(wanted, ev.pools_per_launch(M))
        st = ev.search(m, M)
    assert (st.explored_tree, st.explored_sol) == (171129071, 2279184)  # tests/golden/counts.json
    want, most_rounds = emulated_step2(P, wanted)
    if pools is None:
        assert P > 1 and most_rounds > 2048, "the group loop's call boundary is not exercised"
    got = (st.offloads, st.offloaded_parents, st.per_gpu_tree[0], st.kernel_launches)
    assert got == want

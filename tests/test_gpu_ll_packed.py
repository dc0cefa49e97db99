"""GPU tests of the persistent N-Queens kernel's packed 32-byte pool nodes (nq_rounds_ll.cuh) at the largest boards,
where the packed form uses its whole 125-bit budget, and of the node check that guards it (tsb_nq_pool_push)."""
import numpy as np
import pytest

import tsb200
from test_gpu_parity import rand_nq

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("N,rounds", [(18, 12), (19, 10), (20, 8)])
def test_pool_run_equals_pool_steps_on_large_boards(N, rounds):
    """one pool: the persistent kernel (1, 3, then the rest of the rounds per launch) against the two-kernel rounds on
    the plain 21-byte pool: same counters, byte-identical pools"""
    m, M = 25, 50000
    rng = np.random.default_rng(N * 31 + 7)
    start = rand_nq(rng, N, 60, depth_lo=1, depth_hi=2)
    with tsb200.NQueensEvaluator(N, M=M) as a, tsb200.NQueensEvaluator(N, M=M) as b:
        a.pool_push(start)
        b.pool_push(start)
        tot = [0, 0, 0, 0]
        for _ in range(rounds):
            n_par, n_child, n_sol = a.pool_step(m, M)
            if n_par == 0:
                break
            tot = [tot[0] + 1, tot[1] + n_par, tot[2] + n_child, tot[3] + n_sol]
        assert tot[0] == rounds
        got = [0, 0, 0, 0]
        for k in (1, 3, rounds):
            r = b.pool_run(m, M, min(k, rounds - got[0]))
            got = [x + y for x, y in zip(got, r)]
        assert got == tot and a.pool_size == b.pool_size
        assert a.pool_drain().tobytes() == b.pool_drain().tobytes()


@pytest.mark.parametrize("N,rounds", [(17, 400), (20, 60)])
def test_four_pools_per_launch_equal_separate_pool_runs(N, rounds):
    """four pools in shared launches (two CTAs per SM, 768 parents per CTA: the variant of the N = 17 --M 50000
    search) against each pool run on its own: same counters, byte-identical pools"""
    m, M, K = 25, 50000, 4
    rng = np.random.default_rng(N * 77 + K)
    starts = [rand_nq(rng, N, 40 + 13 * i, depth_lo=1, depth_hi=2) for i in range(K)]
    multi = [tsb200.NQueensEvaluator(N, M=M) for _ in range(K)]
    try:
        assert multi[0].pools_per_launch(M) == K
        for ev, st in zip(multi, starts):
            ev.pool_push(st)
        got = tsb200.nqueens_pool_run_multi(multi, m, M, rounds)
        assert max(x[1] for x in got) > 10 * M  # the pools ran full chunks
        for i, st in enumerate(starts):
            with tsb200.NQueensEvaluator(N, M=M) as one:
                one.pool_push(st)
                assert got[i] == one.pool_run(m, M, rounds)
                assert multi[i].pool_size == one.pool_size
                assert multi[i].pool_drain().tobytes() == one.pool_drain().tobytes()
    finally:
        for ev in multi:
            ev.close()


def test_pool_push_refuses_nodes_the_search_cannot_create():
    """depth > N, a board value >= N, or a nonzero byte past N: TSB_EINVAL, and the pool is unchanged"""
    N = 12
    rng = np.random.default_rng(5)
    good = rand_nq(rng, N, 50, depth_lo=0, depth_hi=N)
    good["depth"][0] = N  # a leaf is a node like any other
    with tsb200.NQueensEvaluator(N, M=1000) as ev:
        ev.pool_push(good)
        for field, row, col, value in (("depth", 7, None, N + 1), ("depth", 7, None, 255), ("board", 3, 5, N),
                                       ("board", 3, 0, 31), ("board", 9, N, 1), ("board", 9, 19, 2)):
            bad = rand_nq(rng, N, 20)
            if col is None:
                bad[field][row] = value
            else:
                bad[field][row, col] = value
            with pytest.raises(tsb200.TsbError):
                ev.pool_push(bad)
            assert ev.pool_size == good.shape[0]
        assert ev.pool_drain().tobytes() == good.tobytes()
        # and the pool still works: a good push after the refused ones, then rounds
        ev.pool_push(good)
        assert ev.pool_run(1, 1000, 5)[1] >= good.shape[0]

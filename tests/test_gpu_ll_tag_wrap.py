"""The 16-bit node tags of the persistent N-Queens kernel (nq_rounds_ll.cuh) over searches of more than 3 x 65 535
rounds, bit-exact against the oracle's pool loop after every call.  A pool's tags are cleared before a launch that
would run out of epochs whose tags cannot alias, and a launch that reaches the last such epoch leaves and is
relaunched.  Covered:
  - launches that start one epoch below the end of the window (no clear, the launch uses exactly its last epoch) and
    at its end (clear first), and calls that cross the end inside one call (relaunch, clear, go on);
  - pools drained and pushed back after every call: the import stores tag 0 and the arena above the pool keeps the
    nodes of earlier rounds and launches;
  - two pools in shared launches whose windows end at different rounds.
N = 12 at M = 4: 214 049 rounds, with the pool rising and falling below 115 nodes."""
import pytest

import tsb200
from test_gpu_nq_boards import Handles, OraclePool, assert_pool, root, run_and_check

pytestmark = pytest.mark.gpu

N, M = 12, 4
SPAN = 65535  # LL_TAG_SPAN: epochs after a clear that a launch may use


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


def test_calls_that_start_at_the_end_of_the_tag_window():
    """a fresh handle's epoch is its round count: the calls end at epochs SPAN - 1 (one left), SPAN (none left: the
    next call clears first), SPAN + 2, then cross 2 SPAN inside a call, and the last call runs the search out across
    3 SPAN; the pool is drained and compared after every call"""
    o = OraclePool(N, root(N))
    with Handles(N, M, 1) as evs:
        evs[0].pool_push(root(N))
        for k in [SPAN - 1, 1, 2, SPAN - 1, 3, 1000, 10 ** 9]:
            run_and_check(evs, [o], 1, M, k)
    assert len(o.rounds) > 3 * SPAN and o.size == 0


@pytest.mark.parametrize("P", [1, 2])
def test_whole_search_in_one_call(P):
    """one call for the whole search: the launches end at the window's last epoch, clear and go on; with two pools
    the second one's window ends 1 000 rounds earlier (it ran those alone first)"""
    oracles = [OraclePool(N, root(N)) for _ in range(P)]
    with Handles(N, M, P) as evs:
        for ev in evs:
            ev.pool_push(root(N))
        if P > 1:
            run_and_check(evs[1:], oracles[1:], 1, M, 1000)
        if P == 1:
            got = [evs[0].pool_run(1, M, 10 ** 9)]
        else:
            got = tsb200.nqueens_pool_run_multi(evs, 1, M, 10 ** 9)
        for ev, o, g in zip(evs, oracles, got):
            assert list(g) == o.run(1, M, 10 ** 9)
            assert_pool(ev, o)
    assert all(len(o.rounds) > 3 * SPAN and o.size == 0 for o in oracles)

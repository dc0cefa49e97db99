"""The round of the persistent N-Queens kernel (nq_rounds_ll.cuh) around its two hand-overs and its list of parents
with children, bit-exact against the oracle's pool loop and against the two-kernel rounds (pool_step), with the oracle
asserting that each shape was reached:
  - launches of 1, 2 and 3 rounds that resume (PAUSE, decided after the handoff, behind LL_BAR_NEXT);
  - one pool running dry (DONE) while the other pools of the launch go on;
  - arena growth (SPACE) inside a multi-pool launch;
  - a long search in one launch, with the depth bound on the layer stack that keeps RELAUNCH out of reach;
  - chunk sizes that change from round to round (tail rounds below M, chunks of fewer than 2G parents), so that the
    kept sub-slice geometry is recomputed;
  - slices where no parent, every parent, or only the last parent of each worker thread has children.
Each case runs at 1, 2 and 4 pools per launch."""
import numpy as np
import pytest

from test_gpu_nq_boards import (LL_T, Handles, OraclePool, assert_pool, child_counts, ll_grid, mixed_nodes,
                                random_nodes, root, run_and_check, sub_slices, var2_M)

pytestmark = pytest.mark.gpu

POOLS = [1, 2, 4]
LL_LAYERS = 1024  # nq_rounds_ll.cuh


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


@pytest.fixture(scope="module")
def sms():
    import tsb200
    n = int(tsb200.lib().tsb_device_sm_count(0))
    assert n > 0
    return n


def chunk_limit(sms, P, small):
    """M for P pools: `small` (one or two pools) or the four-pool tier's 3-parents-per-thread variant"""
    return small if P < 4 else var2_M(sms, P)


def check_pool_step(N, start, o, m, M):
    """the two-kernel rounds from the same start: every round of the oracle, and its pool at the end"""
    import tsb200
    with tsb200.NQueensEvaluator(N, M=M) as ev:
        ev.pool_push(start)
        for r in o.rounds:
            assert ev.pool_step(m, M) == (r["parents"], r["children"], r["solutions"])
        assert ev.pool_size == o.size
        assert ev.pool_drain().tobytes() == o.pool.tobytes()


def run_group(N, starts, m, M, rounds_per_launch):
    """all pools in shared launches of up to rounds_per_launch[i] rounds each, against the oracle and pool_step;
    the oracles"""
    oracles = [OraclePool(N, s) for s in starts]
    with Handles(N, M, len(starts)) as evs:
        for ev, s in zip(evs, starts):
            ev.pool_push(s)
        for k in rounds_per_launch:
            run_and_check(evs, oracles, m, M, k)
    for s, o in zip(starts, oracles):
        check_pool_step(N, s, o, m, M)
    return oracles


@pytest.mark.parametrize("N", [12, 17])
@pytest.mark.parametrize("P", POOLS)
def test_pause_after_one_two_three_rounds(N, P, sms):
    """every launch ends by PAUSE after 1, 2 or 3 rounds and the next one resumes where it stopped"""
    M = chunk_limit(sms, P, 6000)
    rng = np.random.default_rng(9700 + 10 * N + P)
    starts = [np.concatenate([mixed_nodes(rng, N, 2 * M), random_nodes(rng, N, M + 37 * i, depth_lo=N - 6,
                                                                        depth_hi=N - 3)]) for i in range(P)]
    oracles = run_group(N, starts, 1, M, [1, 2, 3, 3, 2, 1])
    assert all(len(o.rounds) == 12 and o.size >= 1 for o in oracles)


@pytest.mark.parametrize("N", [12, 17])
@pytest.mark.parametrize("P", [2, 4])
def test_one_pool_done_while_the_others_run(N, P, sms):
    """pool 0 runs dry (DONE) after a few rounds; the others keep running in the same launch"""
    M = chunk_limit(sms, P, 6000)
    m = 25
    rng = np.random.default_rng(9800 + 10 * N + P)
    starts = [random_nodes(rng, N, 60, depth_lo=N - 2, depth_hi=N)] + \
             [np.concatenate([mixed_nodes(rng, N, 3 * M), random_nodes(rng, N, M, depth_lo=N - 6, depth_hi=N - 4)])
              for _ in range(P - 1)]
    oracles = run_group(N, starts, m, M, [12])
    assert oracles[0].size < m and len(oracles[0].rounds) < 12
    assert all(len(o.rounds) == 12 for o in oracles[1:])


@pytest.mark.parametrize("N", [12, 17])
@pytest.mark.parametrize("P", [2, 4])
def test_arena_growth_inside_a_multi_pool_launch(N, P, sms, monkeypatch):
    """a small arena: a pool leaves the shared launch for room (SPACE), grows and comes back in a fresh launch"""
    cap = 4000
    monkeypatch.setenv("TSB200_POOL_CAP", str(cap))
    M = chunk_limit(sms, P, 6000)
    rng = np.random.default_rng(9900 + 10 * N + P)
    starts = [random_nodes(rng, N, 200, depth_lo=N - 6, depth_hi=N - 3)] + \
             [random_nodes(rng, N, 40, depth_lo=N - 3, depth_hi=N) for _ in range(P - 1)]
    oracles = run_group(N, starts, 1, M, [10 ** 9])
    need = [[x["s0"] + x["parents"] * N for x in o.rounds] for o in oracles]
    assert all(n[0] <= cap for n in need)
    assert max(need[0][1:]) > cap


class PeakLayers(OraclePool):
    """the oracle's pool loop, recording the most layers the kernel's layer stack held after any round"""
    peak = 0

    def step(self, m, M):
        r = super().step(m, M)
        self.peak = max(self.peak, len(self.layers))
        return r


@pytest.mark.parametrize("P", POOLS)
def test_long_search_and_the_layer_stack(P, sms):
    """whole searches in ONE launch (N = 11 at M = 20, or N = 14 from the root at the four-pool M: hundreds of rounds
    each).  The layer stack grows only while a round has more children than the next chunk takes, and the nodes above
    a surviving layer all descend from it, so the layers' smallest depths strictly increase: at most N + 2 layers,
    far below the LL_LAYERS entries whose end would make the kernel leave for a relaunch.  The oracle checks the
    bound on every round."""
    N, M = (11, 20) if P < 4 else (14, var2_M(sms, P))
    rng = np.random.default_rng(10000 + P)
    starts = [random_nodes(rng, N, 30 + 7 * i, depth_lo=2, depth_hi=4) for i in range(P)]
    if P == 4:
        starts[0] = root(N)
    oracles = [PeakLayers(N, s) for s in starts]
    with Handles(N, M, P) as evs:
        for ev, s in zip(evs, starts):
            ev.pool_push(s)
        run_and_check(evs, oracles, 1, M, 10 ** 9)
    assert all(o.size == 0 for o in oracles)
    assert max(len(o.rounds) for o in oracles) > 300
    assert 3 <= max(o.peak for o in oracles) <= N + 2 < LL_LAYERS
    for s, o in zip(starts, oracles):
        check_pool_step(N, s, o, 1, M)


@pytest.mark.parametrize("N", [12, 17])
@pytest.mark.parametrize("P", POOLS)
def test_chunk_size_changes_between_rounds(N, P, sms):
    """chunks of M, then tail rounds below M and back to M, and chunks of fewer than 2G parents: the sub-slices kept
    from the previous round are recomputed whenever the chunk's size changes"""
    M = chunk_limit(sms, P, 6000)
    G, _ = ll_grid(sms, M, P)
    rng = np.random.default_rng(10100 + 10 * N + P)
    # [M + a few shallow-ish nodes][M deep nodes]: rounds of M, then the pool shrinks below M (tail rounds), and the
    # shallow nodes below bring chunks of M back
    starts = [np.concatenate([random_nodes(rng, N, M // 3 + 11 * i, depth_lo=N - 8, depth_hi=N - 7),
                              random_nodes(rng, N, M + 5 * i, depth_lo=N - 2, depth_hi=N)]) for i in range(P)]
    small = [random_nodes(rng, N, G + 3 + i, depth_lo=N - 4, depth_hi=N - 2) for i in range(P)]
    oracles = run_group(N, starts, 1, M, [40])
    for o in oracles:
        n = [x["parents"] for x in o.rounds]
        assert n[0] == M and any(a == M and b < M for a, b in zip(n, n[1:]))
        assert any(a < M and b == M for a, b in zip(n, n[1:]))
    oracles = run_group(N, small, 1, M, [40])
    for o in oracles:
        n = [x["parents"] for x in o.rounds]
        assert any(x < 2 * G for x in n) and len(set(n)) > 2


def thread_slots(n, G, ppt):
    """(CTA, worker thread, parent of the thread) of every chunk position, for a chunk of n parents"""
    where = np.zeros((n, 3), dtype=np.int64)
    for k, (a0, l0, a1, l1) in enumerate(sub_slices(n, G)):
        for i in range(l0 + l1):
            pos = a0 + i if i < l0 else a1 + (i - l0)
            where[pos] = (k, i // ppt, i % ppt)
    return where


@pytest.mark.parametrize("N", [12, 17])
@pytest.mark.parametrize("P", POOLS)
def test_parents_with_children_lists(N, P, sms):
    """round 1 of each pool is a whole pool of M parents where no parent (leaves and dead ends), every parent (depth 0
    and 1), or only the last parent of each worker thread (depth 1 among leaves) has children"""
    M = chunk_limit(sms, P, 6000)
    G, ppt = ll_grid(sms, M, P)
    assert G * LL_T * ppt >= M
    rng = np.random.default_rng(10200 + 10 * N + P)
    where = thread_slots(M, G, ppt)
    last = where[:, 2] == ppt - 1

    def none():
        x = random_nodes(rng, N, M, depth_lo=N)
        dead = random_nodes(rng, N, 8 * M, depth_lo=N - 2, depth_hi=N - 1)
        dead = dead[child_counts(dead, N) == 0]
        assert dead.shape[0] >= M // 2
        x[1::2] = dead[:x[1::2].shape[0]]
        return x

    def every():
        return random_nodes(rng, N, M, depth_lo=0, depth_hi=1)

    def last_only():
        x = random_nodes(rng, N, M, depth_lo=N)
        x[last] = random_nodes(rng, N, int(last.sum()), depth_lo=1, depth_hi=1)
        return x

    kinds = [none, every, last_only]
    for i in range(0, 3, P) if P < 3 else [0]:
        group = [kinds[(i + j) % 3]() for j in range(P)]
        want = [kinds[(i + j) % 3] for j in range(P)]
        for w, s in zip(want, group):
            cc = child_counts(s, N)
            if w is none:
                assert (cc == 0).all()
            elif w is every:
                assert (cc > 0).all()
            else:
                assert ((cc > 0) == last).all() and last.any() and not last.all()
        run_group(N, group, 1, M, [1, 1])

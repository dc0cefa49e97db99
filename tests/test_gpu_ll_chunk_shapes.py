"""Where the next round's chunk lies relative to a round's children, for the persistent N-Queens kernel
(nq_rounds_ll.cuh), bit-exact against the oracle's pool loop, with the oracle asserting that each shape was reached:
  - fewer children than the next chunk: it reaches below them into older layers, from inside one of its sub-slices
    and over several of them;
  - more children than the next chunk: the bottom children stay below it;
  - one CTA with more than 2 LL_CAP children, whose children span several of the next round's sub-slices;
  - a round without children; next chunks of fewer than 2G parents (empty sub-slices);
  - launches that stop after 1, 2 and 3 rounds and resume;
  - arena growth (a pool leaves a four-pool launch for room and comes back).
Each case runs at 1, 2 and 4 pools per launch and at N = 12, 17, 20 (the dense case at 17 and 20)."""
import numpy as np
import pytest

from test_gpu_nq_boards import (LL_CAP, Handles, OraclePool, child_counts, dense_shares, ll_grid, mixed_nodes,
                                random_nodes, run_and_check, sub_slices, var2_M, zero_children_pool)

pytestmark = pytest.mark.gpu

BOARDS = [12, 17, 20]
POOLS = [1, 2, 4]


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


def run_group(N, starts, m, M, rounds_per_launch):
    """all pools in shared launches of up to rounds_per_launch[i] rounds each, against the oracle; the oracles"""
    oracles = [OraclePool(N, s) for s in starts]
    with Handles(N, M, len(starts)) as evs:
        for ev, s in zip(evs, starts):
            ev.pool_push(s)
        for k in rounds_per_launch:
            run_and_check(evs, oracles, m, M, k)
    return oracles


def next_chunks(o, M):
    """per round: (children, n' = the next round's chunk, the round's own s0, the next s0)"""
    out = []
    for a, b in zip(o.rounds, o.rounds[1:]):
        out.append((a["children"], b["parents"], a["s0"], b["s0"]))
    return out


def group_of(P, make):
    return [make(i) for i in range(P)]


@pytest.mark.parametrize("N", BOARDS)
@pytest.mark.parametrize("P", POOLS)
def test_next_chunk_reaches_below_the_children(N, P, sms):
    """[older nodes][M deep nodes]: the rounds produce fewer children than M, so the next chunk starts below them,
    inside a sub-slice of the next round and over several of them"""
    M = chunk_limit(sms, P, 6000)
    G, _ = ll_grid(sms, M, P)
    rng = np.random.default_rng(9100 + 10 * N + P)
    starts = group_of(P, lambda i: np.concatenate([mixed_nodes(rng, N, 3 * M),
                                                   random_nodes(rng, N, M, depth_lo=N - 4, depth_hi=N - 2)]))
    oracles = run_group(N, starts, 1, M, [4])
    for o in oracles:
        below = [(c, n1, s0, s01) for c, n1, s0, s01 in next_chunks(o, M) if c < n1]
        assert below
        # the older part of the next chunk covers more than two of its sub-slices, and its top is not a sub-slice start
        deep = [(s0 - s01, n1) for c, n1, s0, s01 in below]
        assert any(x > 2 * n1 // (2 * G) for x, n1 in deep)
        assert any(all(x != n1 * j // (2 * G) for j in range(2 * G + 1)) for x, n1 in deep)


@pytest.mark.parametrize("N", BOARDS)
@pytest.mark.parametrize("P", POOLS)
def test_children_beyond_the_next_chunk(N, P, sms):
    """shallow parents: a round has more children than M, its bottom children stay below the next chunk"""
    M = chunk_limit(sms, P, 6000)
    rng = np.random.default_rng(9200 + 10 * N + P)
    starts = group_of(P, lambda i: random_nodes(rng, N, M + 17 * i, depth_lo=2, depth_hi=4))
    oracles = run_group(N, starts, 1, M, [3])
    for o in oracles:
        assert any(c > n1 and n1 == M for c, n1, _, _ in next_chunks(o, M))


@pytest.mark.parametrize("N", [17, 20])
@pytest.mark.parametrize("P", POOLS)
def test_a_range_spans_several_next_sub_slices(N, P, sms):
    """depth 0 / 1 parents: a CTA's share has more than 2 LL_CAP children (several staging windows), and its children
    span several sub-slices of the next round"""
    M = chunk_limit(sms, P, 40000)
    G, _ = ll_grid(sms, M, P)
    rng = np.random.default_rng(9300 + 10 * N + P)
    starts = [random_nodes(rng, N, M, depth_lo=0, depth_hi=1)] + [random_nodes(rng, N, 500 + 31 * i, depth_lo=N - 3)
                                                                  for i in range(P - 1)]
    shares = dense_shares(starts[0], N, G)
    assert max(s for s, _ in shares) > 2 * LL_CAP
    o = run_group(N, starts, 1, M, [2])[0]
    # the children of the top sub-slice (CTA 0's) that lie inside the next chunk cover more than two of its sub-slices
    cc = child_counts(starts[0], N)
    a1, l1 = sub_slices(M, G)[0][2:]
    n1 = o.rounds[1]["parents"]
    top = cc[a1:a1 + l1].sum()
    assert min(top, n1) > 2 * (n1 // (2 * G))


@pytest.mark.parametrize("N", BOARDS)
@pytest.mark.parametrize("P", POOLS)
def test_zero_children_and_tiny_next_chunks(N, P, sms):
    """a round without children (the next one reads older nodes only), and next chunks of fewer than 2G parents"""
    M = chunk_limit(sms, P, 3001)
    G, _ = ll_grid(sms, M, P)
    rng = np.random.default_rng(9400 + 10 * N + P)
    starts = group_of(P, lambda i: zero_children_pool(rng, N, M) if i % 2 == 0 else
                      random_nodes(rng, N, G + 5 * i, depth_lo=N - 3, depth_hi=N - 1))
    oracles = run_group(N, starts, 1, M, [8])
    assert any(x["children"] == 0 for x in oracles[0].rounds[:-1])
    if P > 1:
        assert any(r["parents"] < 2 * G for r in oracles[1].rounds[1:])


@pytest.mark.parametrize("N", BOARDS)
@pytest.mark.parametrize("P", POOLS)
def test_launches_of_one_two_three_rounds(N, P, sms):
    """launches that stop after 1, 2 and 3 rounds (PAUSE) and resume: every launch starts with one trusted layer"""
    M = chunk_limit(sms, P, 6000)
    rng = np.random.default_rng(9500 + 10 * N + P)
    starts = group_of(P, lambda i: np.concatenate([mixed_nodes(rng, N, 2 * M),
                                                   random_nodes(rng, N, M // 2 + 101 * i, depth_lo=N - 6,
                                                                depth_hi=N - 3)]))
    oracles = run_group(N, starts, 1, M, [1, 2, 3, 1, 2, 3])
    assert all(len(o.rounds) == 12 for o in oracles)


@pytest.mark.parametrize("N", BOARDS)
def test_arena_growth_inside_a_four_pool_launch(N, sms, monkeypatch):
    """a small arena: pools leave the shared launch for room (SPACE), grow and come back in a fresh launch"""
    cap = 4000
    monkeypatch.setenv("TSB200_POOL_CAP", str(cap))
    M = var2_M(sms, 4)
    rng = np.random.default_rng(9600 + N)
    starts = [random_nodes(rng, N, 30, depth_lo=N - 5, depth_hi=N - 4),
              random_nodes(rng, N, 40, depth_lo=N - 3, depth_hi=N),
              random_nodes(rng, N, 200, depth_lo=N - 6, depth_hi=N - 3),
              random_nodes(rng, N, 10, depth_lo=N - 3, depth_hi=N)]
    oracles = run_group(N, starts, 1, M, [10 ** 9])
    need = [[x["s0"] + x["parents"] * N for x in o.rounds] for o in oracles]
    assert all(n[0] <= cap for n in need)
    assert any(max(n[1:], default=0) > cap for n in need)

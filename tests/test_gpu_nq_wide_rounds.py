"""The persistent N-Queens kernel on wide handles (tsb_nq_create_wide: 25-byte records, nq_rounds_ll_wide_kernel, one
pool per launch), bit-exact against the oracle built with OR_MAX_QUEENS = 24 (oracle/pyoracle24): every call's
counters and the pool byte for byte after it.  A wide fat node stores board[18..23] where a 20-queen node keeps its
child mask and leaf flag, so the kernel evaluates a parent's child mask when it reads it.  Covered:
  - the route: pool_run takes the persistent kernel (a handful of launches for any number of rounds) up to the one-pool
    capacity and two-kernel rounds beyond it or under TSB200_NO_ROUNDS=1, with the same results and pools, on the
    N = 21..24 subtrees of tests/golden/nqueens_wide.json (their tree and solution counts);
  - every N = 1..24, and at the kernel's edges (the one-pool cases of test_gpu_nq_boards.py and
    test_gpu_ll_chunk_shapes.py): next chunks below and above a round's children, rounds without children, chunks over
    several layers, launches of 1, 2 and 3 rounds, full slices at the one-pool capacity and one past it, arena growth,
    CTAs whose children need several staging windows (up to 24 children per parent);
  - the 16-bit tag window over more than 3 x 65 535 rounds;
  - a steal between two wide handles straight after persistent launches;
  - whole searches on the wide route with far fewer kernel launches than rounds."""
import json
import os

import numpy as np
import pytest

import tsb200
from oracle import pyoracle24 as po24
from test_gpu_nq_boards import LL_CAP, OraclePool, assert_pool, ll_grid, pool_capacity, sub_slices
from test_gpu_nq_wide import goldens, subtree_root

pytestmark = pytest.mark.gpu
W = tsb200.NQ_NODE24_DTYPE
BOARDS = list(range(1, 25))
EDGE_BOARDS = [5, 12, 17, 20, 21, 22, 23, 24]
SHAPE_BOARDS = EDGE_BOARDS[1:]  # (boards with enough children per node for the chunk shapes below)
SPAN = 65535  # LL_TAG_SPAN


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


@pytest.fixture(scope="module")
def sms():
    n = int(tsb200.lib().tsb_device_sm_count(0))
    assert n > 0
    return n


# ------------------------------------------------------------------------------------------ nodes and the oracle
def random_nodes(rng, N, count, depth_lo=0, depth_hi=None):
    """random boards (row-wise permutations of 0..N-1) at random depths, bytes past N zero"""
    depth_hi = N if depth_hi is None else depth_hi
    nodes = np.zeros(count, dtype=W)
    nodes["depth"] = rng.integers(max(0, depth_lo), depth_hi + 1, size=count)
    nodes["board"][:, :N] = np.argsort(rng.random((count, N)), axis=1).astype(np.uint8)
    return nodes


def mixed_nodes(rng, N, count):
    """random depths with roots (depth 0) and leaves (depth N) among them"""
    nodes = random_nodes(rng, N, count)
    nodes["depth"][0::7] = 0
    nodes["depth"][3::7] = N
    return nodes


def deep_nodes(rng, N, count):
    """nodes with few children: depths N - 3 .. N"""
    return random_nodes(rng, N, count, depth_lo=N - 3, depth_hi=N)


def root(N):
    r = np.zeros(1, dtype=W)
    r["board"][0, :N] = np.arange(N)
    return r


def child_counts(nodes, N):
    """children of every node: its live slots the oracle labels safe (none for a leaf)"""
    lab = po24.nq_evaluate(np.ascontiguousarray(nodes), N).reshape(-1, N)
    live = np.arange(N)[None, :] >= nodes["depth"][:, None].astype(np.int64)
    return ((lab == 1) & live).sum(axis=1)


class WidePool(OraclePool):
    """test_gpu_nq_boards.OraclePool on 25-byte records: the oracle's rounds as a MAX_QUEENS = 24 build runs them"""

    def __init__(self, N, nodes):
        self.N = N
        self.pool = np.ascontiguousarray(nodes, dtype=W).copy()
        self.rounds = []
        self.launch()

    def step(self, m, M):
        size = self.size
        if size < m:
            return None
        n = min(size, M)
        s0 = size - n
        ends = self.layers[1:] + [size]
        spanned = sum(1 for b, e in zip(self.layers, ends) if e > s0)
        chunk = np.ascontiguousarray(self.pool[s0:])
        kids, sol = po24.nq_expand(chunk, self.N)
        self.layers = [b for b in self.layers if b < s0] + ([s0] if kids.shape[0] else [])
        self.pool = np.concatenate([self.pool[:s0], kids.view(W)])
        r = dict(parents=n, children=kids.shape[0], solutions=sol, s0=s0, layers=spanned, chunk=chunk)
        self.rounds.append(r)
        return r

    def steal_to(self, thief, m):
        """tsb_nq_pool_steal: the oldest half of a pool of at least 2 m nodes"""
        if self.size < 2 * m:
            return 0
        k = self.size // 2
        thief.pool = np.concatenate([thief.pool, self.pool[:k]])
        self.pool = self.pool[k:].copy()
        return k


def wide(N, M):
    ev = tsb200.NQueensEvaluator(N, M=M, max_queens=24)
    assert ev.wide and ev.pools_per_launch(M) == 1
    return ev


def run_and_check(ev, o, m, M, max_rounds):
    """one pool_run call against the oracle's loop: counters and pool; -> the call's kernel launches"""
    l0 = ev.kernel_launches
    got = ev.pool_run(m, M, max_rounds)
    launches = ev.kernel_launches - l0
    assert list(got) == o.run(m, M, max_rounds)
    assert_pool(ev, o)
    return launches


def run_group(N, start, m, M, calls):
    """one wide pool, one pool_run call per entry of `calls` (its round budget), checked after each; the oracle"""
    o = WidePool(N, start)
    with wide(N, M) as ev:
        ev.pool_push(start)
        for k in calls:
            launches = run_and_check(ev, o, m, M, k)
            # the persistent kernel: the import, one launch (two at a tag clear) and the export of the drain
            assert launches <= 4, (k, launches)
    return o


def next_chunks(o):
    """per round: (children, n' = the next round's chunk, the round's own s0, the next s0)"""
    return [(a["children"], b["parents"], a["s0"], b["s0"]) for a, b in zip(o.rounds, o.rounds[1:])]


# ------------------------------------------------------------------------------------------ the route
def pool_run_calls(N, prefix, M, calls, no_rounds, monkeypatch):
    """the subtree of `prefix` in pool_run calls of `calls` rounds each; per call: (counters, launches, the pool)"""
    if no_rounds:
        monkeypatch.setenv("TSB200_NO_ROUNDS", "1")
    else:
        monkeypatch.delenv("TSB200_NO_ROUNDS", raising=False)
    out = []
    with wide(N, M) as ev:
        ev.pool_push(subtree_root(N, prefix))
        for k in calls:
            l0 = ev.kernel_launches
            got = tuple(ev.pool_run(1, M, k))
            launches = ev.kernel_launches - l0
            pool = ev.pool_drain()
            if pool.shape[0]:
                ev.pool_push(pool)
            out.append((got, launches, pool.tobytes()))
    return out


@pytest.mark.parametrize("M", [50000, 2000])
@pytest.mark.parametrize("s", range(8))
def test_route_persistent_against_two_kernel_rounds(s, M, golden_dir, monkeypatch):
    """the persistent kernel takes a handful of launches per call for any number of rounds, the two-kernel rounds at
    least two per round; both give the same counters and pools after every call, and the subtree's golden counts"""
    g = goldens(golden_dir)[s]
    calls = [1, 2, 40, 10 ** 9]
    ll = pool_run_calls(g["N"], g["prefix"], M, calls, False, monkeypatch)
    steps = pool_run_calls(g["N"], g["prefix"], M, calls, True, monkeypatch)
    for (got, launches, pool), (want, step_launches, want_pool) in zip(ll, steps):
        assert got == want and pool == want_pool
        assert launches <= 6 and step_launches >= 2 * want[0]
    rounds, parents, children, sols = (sum(x[0][i] for x in ll) for i in range(4))
    assert (children, sols) == (g["tree"], g["sol"]) and parents == g["tree"] + 1
    assert rounds > 10 and len(ll[-1][2]) == 0


# ------------------------------------------------------------------------------------------ every board size
def start_pool(N, rng):
    """(start nodes, m, M, max rounds): N <= 13 until the pool is empty (m = 1), larger boards a bounded run"""
    if N <= 10:
        return root(N), 1, (7 if N <= 6 else 97 if N <= 9 else 1500), 10 ** 9
    if N <= 13:
        return random_nodes(rng, N, 40, depth_lo=N - 7, depth_hi=N - 4), 1, 1500, 10 ** 9
    return random_nodes(rng, N, 300, depth_lo=2, depth_hi=N), 25, 3000, 24


@pytest.mark.parametrize("N", BOARDS)
def test_pool_run_every_board(N, sms):
    start, m, M, R = start_pool(N, np.random.default_rng(11500 + N))
    assert ll_grid(sms, M, 1)[0] > 0
    o = WidePool(N, start)
    with wide(N, M) as ev:
        ev.pool_push(start)
        done = 0
        for k in (0, 1, 3, R):
            k = min(k, R - done)
            run_and_check(ev, o, m, M, k)
            done += k
    if N <= 13:
        assert o.size == 0
    assert len(o.rounds) > 1


@pytest.mark.parametrize("N", SHAPE_BOARDS)
def test_next_chunk_reaches_below_the_children(N, sms):
    """[older nodes][M deep nodes]: fewer children than M, the next chunk starts below them, inside a sub-slice of the
    next round and over several of them"""
    M = 6000
    G, _ = ll_grid(sms, M, 1)
    rng = np.random.default_rng(11630 + N)
    start = np.concatenate([mixed_nodes(rng, N, 3 * M), random_nodes(rng, N, M, depth_lo=N - 4, depth_hi=N - 2)])
    o = run_group(N, start, 1, M, [4])
    below = [(c, n1, s0, s01) for c, n1, s0, s01 in next_chunks(o) if c < n1]
    assert below
    deep = [(s0 - s01, n1) for c, n1, s0, s01 in below]
    assert any(x > 2 * n1 // (2 * G) for x, n1 in deep)
    assert any(all(x != n1 * j // (2 * G) for j in range(2 * G + 1)) for x, n1 in deep)


@pytest.mark.parametrize("N", SHAPE_BOARDS)
def test_children_beyond_the_next_chunk(N):
    """shallow parents: more children than M, the bottom children stay below the next chunk"""
    M = 6000
    start = random_nodes(np.random.default_rng(11700 + N), N, M, depth_lo=2, depth_hi=4)
    o = run_group(N, start, 1, M, [3])
    assert any(c > n1 and n1 == M for c, n1, _, _ in next_chunks(o))


def zero_children_pool(rng, N, M):
    """[older nodes][M leaves][M nodes of depth N - 1]: round 2 pops leaves only (no children); round 3 reads the
    launch's trusted layer"""
    return np.concatenate([mixed_nodes(rng, N, 3 * M), random_nodes(rng, N, M, depth_lo=N),
                           random_nodes(rng, N, M, depth_lo=N - 1, depth_hi=N - 1)])


def layered_pool(rng, N, M):
    """[older nodes][M parents of depth d]: rounds whose children shrink from more than M to fewer, so that a chunk
    reads the newest layer, the rest of an older round's children and the launch's trusted layer"""
    d = {5: 1, 12: 6, 17: 10, 20: 12, 21: 13, 22: 14, 23: 15, 24: 16}[N]
    return np.concatenate([mixed_nodes(rng, N, 2 * M), random_nodes(rng, N, M, depth_lo=d, depth_hi=d)])


@pytest.mark.parametrize("N", EDGE_BOARDS)
def test_zero_children_rounds_and_chunks_over_several_layers(N, sms):
    M = 3001
    G, _ = ll_grid(sms, M, 1)
    rng = np.random.default_rng(11800 + N)
    o = run_group(N, zero_children_pool(rng, N, M), 1, M, [8])
    zero = [r for r, x in enumerate(o.rounds) if x["children"] == 0]
    assert zero and zero[0] < len(o.rounds) - 1  # a round without children, and rounds after it
    o = run_group(N, layered_pool(rng, N, M), 1, M, [8])
    assert max(x["layers"] for x in o.rounds) >= 3
    # next chunks of fewer than 2G parents (empty sub-slices)
    o = run_group(N, random_nodes(rng, N, G + 5, depth_lo=N - 3, depth_hi=N - 1), 1, M, [8])
    assert any(r["parents"] < 2 * G for r in o.rounds[1:])


@pytest.mark.parametrize("N", EDGE_BOARDS)
def test_launches_of_one_two_three_rounds(N):
    """launches that stop after 1, 2 and 3 rounds (PAUSE) and resume: every launch starts with one trusted layer"""
    M = 6000
    rng = np.random.default_rng(11900 + N)
    start = np.concatenate([mixed_nodes(rng, N, 2 * M), random_nodes(rng, N, M // 2, depth_lo=N - 6, depth_hi=N - 3)])
    o = run_group(N, start, 1, M, [1, 2, 3, 1, 2, 3])
    assert len(o.rounds) == 12


@pytest.mark.parametrize("N", EDGE_BOARDS)
def test_full_slices_and_one_past_the_one_pool_capacity(N, sms, monkeypatch):
    """M = the one-pool capacity: every CTA gets a full slice of 512 parents; M = capacity + 1: two-kernel rounds"""
    cap = pool_capacity(sms, 1)
    rng = np.random.default_rng(12000 + N)
    start = deep_nodes(rng, N, cap + 1 + 97)
    for M in (cap, cap + 1):
        grid, per = ll_grid(sms, M, 1)
        assert (grid * 256 * per == M) if M == cap else grid == 0
        o = WidePool(N, start)
        with wide(N, M) as ev:
            ev.pool_push(start)
            launches = run_and_check(ev, o, 1, M, 2)
        assert o.rounds[0]["parents"] == M
        assert (launches <= 4) if M == cap else launches >= 2 * 2


@pytest.mark.parametrize("N", EDGE_BOARDS)
def test_arena_growth(N, monkeypatch):
    """a small arena (TSB200_POOL_CAP): the pool leaves the launch for room (SPACE), grows and is launched again"""
    cap = 4000
    monkeypatch.setenv("TSB200_POOL_CAP", str(cap))
    rng = np.random.default_rng(12100 + N)
    start = random_nodes(rng, N, 150, depth_lo=N - 6, depth_hi=N - 3)
    o = WidePool(N, start)
    with wide(N, 3001) as ev:
        ev.pool_push(start)
        run_and_check(ev, o, 1, 3001, 10 ** 9)
    need = [x["s0"] + x["parents"] * N for x in o.rounds]
    assert need[0] <= cap and max(need[1:], default=0) > cap


@pytest.mark.parametrize("N", [20, 21, 24])
def test_dense_ctas_use_several_staging_windows(N, sms):
    """depth 0 / 1 parents (a root of a 24-queen board has 24 children): a CTA's share has more than 2 LL_CAP
    children, built in several windows, and a window crosses from the bottom sub-slice's children to the top one's"""
    M = 40000
    G, _ = ll_grid(sms, M, 1)
    rng = np.random.default_rng(12200 + N)
    start = random_nodes(rng, N, M, depth_lo=0, depth_hi=1)
    cc = child_counts(start, N)
    assert cc.max() == N
    shares = [(cc[a0:a0 + l0].sum() + cc[a1:a1 + l1].sum(), cc[a0:a0 + l0].sum()) for a0, l0, a1, l1 in
              sub_slices(M, G)]
    assert min(s for s, _ in shares) > 2 * LL_CAP
    assert any(c0 % LL_CAP and c0 > LL_CAP for _, c0 in shares)
    run_group(N, start, 1, M, [2])


# ------------------------------------------------------------------------------------------ tags, steal, searches
def test_tag_window_over_three_spans():
    """N = 12 at M = 4 on a wide handle: calls that end one epoch before the end of the tag window, at its end, and
    cross it inside a call, until the search has run out (more than 3 x 65 535 rounds)"""
    N, M = 12, 4
    o = WidePool(N, root(N))
    with wide(N, M) as ev:
        ev.pool_push(root(N))
        for k in [SPAN - 1, 1, 2, SPAN - 1, 3, 1000, 10 ** 9]:
            l0 = ev.kernel_launches
            got = ev.pool_run(1, M, k)
            assert list(got) == o.run(1, M, k)
            assert ev.kernel_launches - l0 <= 2 + 2 * (k // (SPAN // 2) + 1)  # (no two-kernel rounds)
            assert_pool(ev, o)
    assert len(o.rounds) > 3 * SPAN and o.size == 0


@pytest.mark.parametrize("N", [21, 24])
def test_steal_after_persistent_launches(N, golden_dir):
    """a steal straight after pool_run (the victim's pool is in the fat arena) and rounds on both pools after it"""
    s = [x for x in goldens(golden_dir) if x["N"] == N][-1]
    m, M = 5, 3000
    victim, thief = WidePool(N, subtree_root(N, s["prefix"])), WidePool(N, np.zeros(0, dtype=W))
    with wide(N, M) as ev, wide(N, M) as th:
        ev.pool_push(subtree_root(N, s["prefix"]))
        assert list(ev.pool_run(1, M, 9)) == victim.run(1, M, 9)
        assert th.pool_steal_from(ev, m) == victim.steal_to(thief, m) > 0
        assert_pool(ev, victim)
        assert_pool(th, thief)
        assert list(th.pool_run(1, M, 5)) == thief.run(1, M, 5)
        assert list(ev.pool_run(1, M, 5)) == victim.run(1, M, 5)
        # and the other way: the thief's pool, in its fat arena, goes back to the victim
        assert ev.pool_steal_from(th, m) == thief.steal_to(victim, m) > 0
        assert_pool(ev, victim)
        assert_pool(th, thief)


@pytest.mark.parametrize("D", [1, 2])
@pytest.mark.parametrize("N", [13, 15])
def test_whole_searches_in_the_persistent_kernel(N, D, golden_dir, monkeypatch):
    """M = 50 000 on the wide route: the counts of counts.json, with far fewer kernel launches than rounds"""
    monkeypatch.delenv("TSB200_NO_ROUNDS", raising=False)
    want = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    st = tsb200.nqueens_search_device(N, 1, 25, 50000, D, max_queens=24)
    assert (st.explored_tree, st.explored_sol) == (want["tree"], want["sol"])
    assert st.offloads > 40 and 0 < st.kernel_launches < st.offloads // 4 + 8 * D

"""Every N-Queens kernel on every board size N = 1..20, bit-exact against the oracle (oracle/tsb_oracle.c), not against
another path of this library: the evaluate kernels (one parent per thread, TMA tile pipeline, its partial last tile),
the fused expand, the device pool's two-kernel rounds (pool_step), the fat-arena import / export and the three
variants of the persistent kernel (nq_rounds_ll.cuh: one pool with 2 parents per thread, two pools with 2, several
pools with 3), at the edges of its launch tiers and of its round structure, and whole searches.

Every size that depends on the GPU (SM count, tier capacities, the small / TMA switch) is derived at run time from
tsb_device_sm_count with the formulas of csrc/ll_tiers.h and nq_ll_grid, so the file holds on any SM count."""
import json
import os

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

BOARDS = list(range(1, 21))
LL_T, LL_CAP, EXP_CAP, NQ_TILE = 256, 2048, 1024, 512  # nq_rounds_ll.cuh, nq_expand.cuh, nq_kernel.cuh
NQ = tsb200.NQ_NODE_DTYPE


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


@pytest.fixture(scope="module")
def sms():
    n = int(tsb200.lib().tsb_device_sm_count(0))
    assert n > 0
    return n


# ------------------------------------------------------------------------------------------ launch tiers
def ctas_per_pool(sms, pools):
    """ll_tiers.h ll_ctas_per_pool"""
    s = min(sms, 256)
    return s if pools <= 1 else 2 * s // pools


def pool_capacity(sms, pools):
    """ll_tiers.h ll_pool_capacity: the largest chunk one launch takes per pool"""
    return ctas_per_pool(sms, pools) * (512 if pools <= 1 else 768)


def ll_grid(sms, M, pools):
    """(CTAs per pool, parents per thread) of the persistent kernel for chunks of up to M parents, as nq_ll_grid
    picks them; CTAs = 0: M is beyond the kernel with this many pools"""
    s = min(sms, 256)
    most = ctas_per_pool(s, pools)
    per = 2 if most * 512 >= M else 3
    grid = max(1, (s * 7 // 8) & ~1) if pools == 1 else most
    while grid * LL_T * per < M and grid < most:
        grid += 1
    ok = M <= grid * LL_T * per and (pools > 1 or per == 2)
    return (grid if ok else 0), per


def variant(sms, M, pools):
    """0: one pool, 2 parents per thread; 1: several pools, 2; 2: several pools, 3 (nq_ll_launch_n)"""
    grid, per = ll_grid(sms, M, pools)
    assert grid > 0
    return 0 if pools == 1 else 1 if per == 2 else 2


def var2_M(sms, pools, extra=4099):
    """a chunk limit that runs `pools` pools in the 3-parents-per-thread variant"""
    M = ctas_per_pool(sms, pools) * 512 + extra
    assert M <= pool_capacity(sms, pools) and variant(sms, M, pools) == 2
    return M


def sub_slices(n, G):
    """the two sub-slices [a0, a0 + len0), [a1, a1 + len1) of each CTA k for a chunk of n parents (step 0)"""
    G2 = 2 * G
    out = []
    for k in range(G):
        a0, a1 = n * k // G2, n * (G2 - 1 - k) // G2
        out.append((a0, n * (k + 1) // G2 - a0, a1, n * (G2 - k) // G2 - a1))
    return out


# ------------------------------------------------------------------------------------------ nodes
def random_nodes(rng, N, count, depth_lo=0, depth_hi=None):
    """random boards (row-wise permutations of 0..N-1) at random depths, bytes past N zero"""
    depth_hi = N if depth_hi is None else depth_hi
    nodes = np.zeros(count, dtype=NQ)
    nodes["depth"] = rng.integers(depth_lo, depth_hi + 1, size=count)
    nodes["board"][:, :N] = np.argsort(rng.random((count, N)), axis=1).astype(np.uint8)
    return nodes


def mixed_nodes(rng, N, count):
    """random depths with roots (depth 0) and leaves (depth N) among them"""
    nodes = random_nodes(rng, N, count)
    nodes["depth"][0::7] = 0
    nodes["depth"][3::7] = N
    return nodes


def root(N):
    r = np.zeros(1, dtype=NQ)
    r["board"][0, :N] = np.arange(N)
    return r


def ov(a):
    return np.ascontiguousarray(a).view(po.NQ_NODE_DTYPE)


def child_counts(nodes, N):
    """children of every node: its live slots the oracle labels safe (none for a leaf)"""
    lab = po.nq_evaluate(ov(nodes), N).reshape(-1, N)
    return ((lab == 1) & po.nq_live_mask(ov(nodes), N)).sum(axis=1)


# ------------------------------------------------------------------------------------------ the oracle's pool loop
class OraclePool:
    """The reference's offload loop on the host: popBackBulk(m, M) -> evaluate + generate_children (po.nq_expand) ->
    children appended.  Each round is recorded as a dict: parents, children, solutions, s0 (the chunk's first
    position), the chunk itself and `layers`, how many layers of the persistent kernel's layer stack the chunk reads.
    The stack follows step 8 of nq_rounds_ll.cuh: a launch starts with one trusted layer (the whole pool); after a
    round every layer that starts inside the chunk is gone and the round's children, if any, form the new top."""

    def __init__(self, N, nodes):
        self.N = N
        self.pool = np.ascontiguousarray(nodes, dtype=NQ).copy()
        self.rounds = []
        self.launch()

    @property
    def size(self):
        return self.pool.shape[0]

    def launch(self):
        self.layers = [0] if self.size else []  # first positions, bottom to top

    def step(self, m, M):
        """one round; None when the pool holds fewer than m nodes"""
        size = self.size
        if size < m:
            return None
        n = min(size, M)
        s0 = size - n
        ends = self.layers[1:] + [size]
        spanned = sum(1 for b, e in zip(self.layers, ends) if e > s0)
        chunk = np.ascontiguousarray(self.pool[s0:])
        kids, sol = po.nq_expand(ov(chunk), self.N)
        self.layers = [b for b in self.layers if b < s0] + ([s0] if kids.shape[0] else [])
        self.pool = np.concatenate([self.pool[:s0], kids.view(NQ)])
        r = dict(parents=n, children=kids.shape[0], solutions=sol, s0=s0, layers=spanned, chunk=chunk)
        self.rounds.append(r)
        return r

    def run(self, m, M, max_rounds):
        """up to max_rounds rounds in one launch: [rounds, parents, children, solutions]"""
        self.launch()
        tot = [0, 0, 0, 0]
        while tot[0] < max_rounds:
            r = self.step(m, M)
            if r is None:
                break
            tot = [tot[0] + 1, tot[1] + r["parents"], tot[2] + r["children"], tot[3] + r["solutions"]]
        return tot


def assert_pool(ev, oracle):
    """the device pool holds the oracle's pool byte for byte; it is pushed back (plain arena) afterwards, so the next
    launch of the persistent kernel imports it again"""
    assert ev.pool_size == oracle.size
    got = ev.pool_drain()
    assert ev.pool_size == 0
    assert got.tobytes() == oracle.pool.tobytes()
    if got.shape[0]:
        ev.pool_push(got)


class Handles:
    def __init__(self, N, M, k):
        self.evs = [tsb200.NQueensEvaluator(N, M=M) for _ in range(k)]

    def __enter__(self):
        return self.evs

    def __exit__(self, *a):
        for ev in self.evs:
            ev.close()


def run_and_check(evs, oracles, m, M, max_rounds):
    """pool_run (one handle) or nqueens_pool_run_multi (several) against the oracle's loop: counters, sizes, pools"""
    if len(evs) == 1:
        got = [evs[0].pool_run(m, M, max_rounds)]
    else:
        got = tsb200.nqueens_pool_run_multi(evs, m, M, max_rounds)
    for ev, o, g in zip(evs, oracles, got):
        assert list(g) == o.run(m, M, max_rounds)
        assert_pool(ev, o)


# ------------------------------------------------------------------------------------------ evaluate
def check_evaluate(ev, nodes, N):
    got = ev.evaluate(nodes).reshape(-1, N)
    want = po.nq_evaluate(ov(nodes), N).reshape(-1, N)
    live = po.nq_live_mask(ov(nodes), N)
    np.testing.assert_array_equal(got[live], want[live])


def tails(N):
    """partial last tiles r with r * 21 and (for N != 16) r * N not multiples of 16: the byte-copy tail of the TMA path"""
    rs = [r for r in range(1, NQ_TILE) if (r * 21) % 16 and ((r * N) % 16 or N == 16)]
    return [3 * NQ_TILE + rs[10], 11 * NQ_TILE + rs[-7]]


@pytest.mark.parametrize("N", BOARDS)
def test_evaluate_small_and_tile_kernels(N, monkeypatch):
    rng = np.random.default_rng(7100 + N)
    with tsb200.NQueensEvaluator(N, M=6000) as ev:  # (fewer than 2 x SMs tiles: the one-parent-per-thread kernel)
        for count in (1, 127, 128, 129, 3001):
            check_evaluate(ev, mixed_nodes(rng, N, count), N)
    monkeypatch.setenv("TSB200_NQ_TILE_THREADS", "128")  # (read when the handle is created: always the TMA kernel)
    with tsb200.NQueensEvaluator(N, M=12 * NQ_TILE) as ev:
        for count in [511, 512, 513] + tails(N):
            check_evaluate(ev, mixed_nodes(rng, N, count), N)


@pytest.mark.parametrize("N", [5, 16, 18, 20])
def test_evaluate_at_the_natural_switch_point(N, sms):
    """2 x SMs x 512 parents: the first count the TMA kernel takes by itself"""
    switch = 2 * sms * NQ_TILE
    rng = np.random.default_rng(7200 + N)
    with tsb200.NQueensEvaluator(N, M=switch + 1) as ev:
        for count in (switch - 1, switch + 1):
            check_evaluate(ev, mixed_nodes(rng, N, count), N)


# ------------------------------------------------------------------------------------------ expand
def check_expand(ev, parents, N):
    got, gsol = ev.expand(parents)
    want, wsol = po.nq_expand(ov(parents), N)
    assert gsol == wsol and got.shape[0] == want.shape[0]
    assert got.tobytes() == want.tobytes()
    return got, gsol


@pytest.mark.parametrize("N", BOARDS)
def test_expand(N):
    rng = np.random.default_rng(7300 + N)
    with tsb200.NQueensEvaluator(N, M=50000) as ev:
        for count in (1, 511, 512, 513):
            check_expand(ev, mixed_nodes(rng, N, count), N)
        # dense: depth 0 / 1 parents, up to N children each; tiles of 512 parents take several passes of the image
        dense = random_nodes(rng, N, 3000, depth_lo=0, depth_hi=min(1, N))
        per_tile = np.add.reduceat(child_counts(dense, N), np.arange(0, 3000, NQ_TILE))
        if N >= 4:
            assert per_tile.max() > EXP_CAP
        check_expand(ev, dense, N)
        # only leaves: no child, every parent a solution
        leaves = random_nodes(rng, N, 700, depth_lo=N)
        got, sol = check_expand(ev, leaves, N)
        assert got.shape[0] == 0 and sol == 700
        # a chunk as the reference's driver hands it to evaluate_gpu (offload #1 of the N-Queens search; the capture
        # runs the whole search on the host, hence only up to N = 14)
        if N <= 14:
            try:
                real = po.nq_capture_chunk(N, 1).view(NQ)
            except IndexError:  # (no such offload: the warm-up finishes the search)
                real = np.zeros(0, dtype=NQ)
            if real.shape[0]:
                check_expand(ev, real, N)


# ------------------------------------------------------------------------------------------ device pool, every N
def start_pool(N, rng):
    """(start nodes, m, M, max rounds): N <= 13 until the pool is empty (m = 1), larger boards a bounded run"""
    if N <= 10:
        return root(N), 1, (7 if N <= 6 else 97 if N <= 9 else 1500), 10 ** 9
    if N <= 13:
        return random_nodes(rng, N, 40, depth_lo=N - 7, depth_hi=N - 4), 1, 1500, 10 ** 9
    return random_nodes(rng, N, 300, depth_lo=2, depth_hi=N), 25, 3000, 24


def start_pools(N, k, seed):
    """k different starts: the base start and the oracle's pool after 1, 2, 3 rounds of it (other sizes and depths,
    so that the pools leave a shared launch at different rounds).  Where that pool holds fewer than m nodes (the
    small boards' searches end within a few rounds), i + 1 copies of the base start instead: every start holds at
    least m nodes, so every pool takes part in the first launch"""
    rng = np.random.default_rng(seed)
    nodes, m, M, R = start_pool(N, rng)
    starts = [nodes]
    o = OraclePool(N, nodes)
    for i in range(1, k):
        o.step(m, M)
        starts.append(o.pool.copy() if o.size >= m else np.concatenate([nodes] * (i + 1)))
    assert all(s.shape[0] >= m for s in starts)
    return starts, m, M, R


@pytest.mark.parametrize("N", BOARDS)
def test_pool_step_round_by_round(N):
    (start,), m, M, R = start_pools(N, 1, 7400 + N)
    o = OraclePool(N, start)
    with tsb200.NQueensEvaluator(N, M=M) as ev:
        ev.pool_push(start)
        for _ in range(min(R, 10 ** 4)):
            r = o.step(m, M)
            got = ev.pool_step(m, M)
            if r is None:
                assert got[0] == 0
                break
            assert got == (r["parents"], r["children"], r["solutions"])
            assert_pool(ev, o)
        assert len(o.rounds) > 1
        if N <= 13:
            assert ev.pool_size == 0


@pytest.mark.parametrize("N", BOARDS)
def test_pool_run_one_pool(N, sms):
    (start,), m, M, R = start_pools(N, 1, 7500 + N)
    assert variant(sms, M, 1) == 0
    o = OraclePool(N, start)
    with tsb200.NQueensEvaluator(N, M=M) as ev:
        ev.pool_push(start)
        done = 0
        for k in (0, 1, 3, R):
            k = min(k, R - done)
            run_and_check([ev], [o], m, M, k)
            done += k
        if N <= 13:
            assert o.size == 0


@pytest.mark.parametrize("N", BOARDS)
@pytest.mark.parametrize("K", [2, 3, 4])
def test_pool_run_multi(N, K, sms):
    """K = 2: two pools, 2 parents per thread; K = 3, 4 (with M above the 2-parent slices): 3 parents per thread"""
    starts, m, M, R = start_pools(N, K, 7600 + 10 * N + K)
    if K > 2:
        M = var2_M(sms, K)
    # the launch takes the pools that hold at least m nodes (rounds_run) and picks its variant by their number:
    # all K pools in the first launch (max_rounds = 1 below)
    assert sum(s.shape[0] >= m for s in starts) == K
    assert variant(sms, M, K) == (1 if K == 2 else 2)
    oracles = [OraclePool(N, s) for s in starts]
    with Handles(N, M, K) as evs:
        for ev, s in zip(evs, starts):
            ev.pool_push(s)
        done = 0
        for k in (0, 1, 3, R):
            k = min(k, R - done)
            run_and_check(evs, oracles, m, M, k)
            done += k
    if N <= 13:
        assert all(o.size == 0 for o in oracles)
        if N >= 5:  # the pools left the shared launch at different rounds
            assert len({len(o.rounds) for o in oracles}) > 1


@pytest.mark.parametrize("N", [12, 17])
@pytest.mark.parametrize("case", ["below_m", "dry"])
def test_pool_run_multi_lone_pool_above_the_one_pool_tier(N, case, sms):
    """M = the one-pool capacity + 1: one launch takes two pools but not one.  A pool left running alone finishes its
    calls in two-kernel rounds, as pool_run runs it: below_m: the other pool holds fewer than m nodes from the start;
    dry: the other pool, a few deep nodes, shares the first call's launch and runs dry in it"""
    M = pool_capacity(sms, 1) + 1
    assert ll_grid(sms, M, 1)[0] == 0 and ll_grid(sms, M, 2)[0] > 0
    m, R = 25, 24
    rng = np.random.default_rng(7650 + N)
    big = random_nodes(rng, N, M + 5000, depth_lo=2, depth_hi=N)
    if case == "below_m":  # (the lone pool is the second handle)
        starts, calls = [deep_nodes(rng, N, m - 1), big], (0, 1, 3, R - 4)
    else:
        starts, calls = [big, deep_nodes(rng, N, 40)], (2, 1, 3, R - 6)
    oracles = [OraclePool(N, s) for s in starts]
    with Handles(N, M, 2) as evs:
        assert evs[0].pools_per_launch(M) == 2
        for ev, s in zip(evs, starts):
            ev.pool_push(s)
        for k in calls:
            run_and_check(evs, oracles, m, M, k)
            if case == "dry":
                assert 1 <= len(oracles[1].rounds) <= 2 and oracles[1].size < m
    lone, other = (oracles[1], oracles[0]) if case == "below_m" else (oracles[0], oracles[1])
    assert len(lone.rounds) == R and all(r["parents"] == M for r in lone.rounds)
    assert other.size < m


# ------------------------------------------------------------------------------------------ persistent-kernel edges
EDGE_BOARDS = [5, 12, 17, 20]


def deep_nodes(rng, N, count):
    """nodes with few children: depths N - 3 .. N"""
    return random_nodes(rng, N, count, depth_lo=max(0, N - 3), depth_hi=N)


@pytest.mark.parametrize("N", EDGE_BOARDS)
@pytest.mark.parametrize("P", [1, 2, 3, 4])
def test_full_slices_and_one_past_the_tier(N, P, sms):
    """M = the tier's capacity: every CTA of every pool gets a full slice (512 or 768 parents, 2 or 3 per thread);
    M = capacity + 1: the launch no longer takes P pools and another path serves them: the same pools"""
    cap = pool_capacity(sms, P)
    rng = np.random.default_rng(7700 + 10 * N + P)
    starts = [deep_nodes(rng, N, cap + 1 + 97 * i) for i in range(P)]
    for M in (cap, cap + 1):
        with Handles(N, M, P) as evs:
            grid, per = ll_grid(sms, M, P)
            if M == cap:
                assert grid * LL_T * per == M  # every CTA full
            else:
                assert grid == 0
            if P > 1:
                assert (evs[0].pools_per_launch(M) >= P) == (M == cap)
            oracles = [OraclePool(N, s) for s in starts]
            for ev, s in zip(evs, starts):
                ev.pool_push(s)
            run_and_check(evs, oracles, 1, M, 2)
            assert all(o.rounds[0]["parents"] == M for o in oracles)


@pytest.mark.parametrize("N", EDGE_BOARDS)
@pytest.mark.parametrize("P", [1, 2, 4])
def test_sub_slice_pairing(N, P, sms):
    """chunks of n < 2G parents (empty sub-slices) and n = +-1 (mod 2G) (sub-slices of unequal length), G = CTAs
    per pool of the variant"""
    M = 20000 if P < 4 else var2_M(sms, P)
    G, _ = ll_grid(sms, M, P)
    sizes = [G // 2 + 1, 2 * G - 1, 2 * G + 1, 6 * G - 1, 8 * G + 1, G + 3, 4 * G + 1, 10 * G - 1]
    rng = np.random.default_rng(7800 + 10 * N + P)
    for i in range(0, len(sizes), P):
        group = sizes[i:i + P]
        assert len(group) == P  # (every launch takes P pools, hence G CTAs per pool)
        starts = [mixed_nodes(rng, N, n) for n in group]
        oracles = [OraclePool(N, s) for s in starts]
        with Handles(N, M, P) as evs:
            for ev, s in zip(evs, starts):
                ev.pool_push(s)
            run_and_check(evs, oracles, 1, M, 3)
        for o, n in zip(oracles, group):
            assert o.rounds[0]["parents"] == n
            assert n < 2 * G or n % (2 * G) in (1, 2 * G - 1)
            lens = [x for s in sub_slices(n, G) for x in (s[1], s[3])]
            assert (0 in lens) if n < 2 * G else (min(lens) < max(lens))


def dense_shares(chunk, N, G):
    """per CTA: (children of its share, children of its bottom sub-slice)"""
    cc = child_counts(chunk, N)
    return [(cc[a0:a0 + l0].sum() + cc[a1:a1 + l1].sum(), cc[a0:a0 + l0].sum()) for a0, l0, a1, l1 in
            sub_slices(chunk.shape[0], G)]


@pytest.mark.parametrize("N", [17, 20])
def test_dense_ctas_use_several_staging_windows(N, sms):
    """depth 0 / 1 parents: a CTA's share has more than LL_CAP children, so its children are built in several windows,
    and a window crosses from the bottom sub-slice's children to the top one's (step 7, dst0 / dst1)"""
    rng = np.random.default_rng(7900 + N)
    for P, M in ((1, 40000), (4, var2_M(sms, 4))):
        G, _ = ll_grid(sms, M, P)
        starts = [random_nodes(rng, N, M, depth_lo=0, depth_hi=1)] + [deep_nodes(rng, N, 500 + 31 * i)
                                                                      for i in range(P - 1)]
        shares = dense_shares(starts[0], N, G)
        assert min(s for s, _ in shares) > 2 * LL_CAP
        assert any(c0 % LL_CAP and c0 > LL_CAP for _, c0 in shares)  # a later window holds both sub-slices' children
        oracles = [OraclePool(N, s) for s in starts]
        with Handles(N, M, P) as evs:
            for ev, s in zip(evs, starts):
                ev.pool_push(s)
            run_and_check(evs, oracles, 1, M, 2)


def zero_children_pool(rng, N, M):
    """[older nodes][M leaves][M nodes of depth N - 1]: round 1 turns the top into leaves (fewer than M), round 2
    pops leaves only (its own children and older ones): no children; round 3 reads the launch's trusted layer"""
    return np.concatenate([mixed_nodes(rng, N, 3 * M), random_nodes(rng, N, M, depth_lo=N),
                           random_nodes(rng, N, M, depth_lo=N - 1, depth_hi=N - 1)])


def layered_pool(rng, N, M):
    """[older nodes][M parents of depth d]: rounds whose children shrink from more than M to fewer, so that a chunk
    reads the newest layer, the rest of an older round's children and the launch's trusted layer"""
    d = {5: 1, 12: 6, 17: 10, 20: 12}[N]
    return np.concatenate([mixed_nodes(rng, N, 2 * M), random_nodes(rng, N, M, depth_lo=d, depth_hi=d)])


@pytest.mark.parametrize("N", EDGE_BOARDS)
@pytest.mark.parametrize("P", [1, 2, 4])
def test_zero_children_rounds_and_chunks_over_several_layers(N, P, sms):
    M = 3001 if P < 4 else var2_M(sms, P)
    rng = np.random.default_rng(8000 + 10 * N + P)
    starts = [zero_children_pool(rng, N, M) if i % 2 == 0 else layered_pool(rng, N, M) for i in range(P)]
    if P == 1:
        starts.append(layered_pool(rng, N, M))
    for i in range(0, len(starts), P):
        group = starts[i:i + P]
        oracles = [OraclePool(N, s) for s in group]
        with Handles(N, M, len(group)) as evs:
            for ev, s in zip(evs, group):
                ev.pool_push(s)
            run_and_check(evs, oracles, 1, M, 8)
        for j, o in enumerate(oracles):
            if (i + j) % 2 == 0:
                zero = [r for r, x in enumerate(o.rounds) if x["children"] == 0]
                assert zero and zero[0] < len(o.rounds) - 1  # a round without children, and rounds after it
            else:
                assert max(x["layers"] for x in o.rounds) >= 3


@pytest.mark.parametrize("N", [12, 17])
def test_arena_growth_inside_a_four_pool_launch(N, sms, monkeypatch):
    """a small arena (TSB200_POOL_CAP, read when a pool is set up): some pools run out of room inside the shared
    launch and are relaunched with fewer pools (another variant and grid) while the others have finished"""
    cap = 4000
    monkeypatch.setenv("TSB200_POOL_CAP", str(cap))
    M = var2_M(sms, 4)
    rng = np.random.default_rng(8100 + N)
    starts = [random_nodes(rng, N, 30, depth_lo=N - 5, depth_hi=N - 4), deep_nodes(rng, N, 40),
              random_nodes(rng, N, 200, depth_lo=N - 6, depth_hi=N - 3), deep_nodes(rng, N, 10)]
    oracles = [OraclePool(N, s) for s in starts]
    with Handles(N, M, 4) as evs:
        for ev, s in zip(evs, starts):
            ev.pool_push(s)
        run_and_check(evs, oracles, 1, M, 10 ** 9)
    # room a round needs before it starts (the kernel's worst case: every slot of every parent survives)
    need = [[x["s0"] + x["parents"] * N for x in o.rounds] for o in oracles]
    # every pool's first round fits the arena: all four pools enter the first launch as they are, nothing grows before
    assert all(n[0] <= cap for n in need)
    # a later round of some pool does not fit: that pool leaves the launch for room (RND_EXIT_SPACE), grows and goes
    # again ...
    assert any(max(n[1:], default=0) > cap for n in need)
    # ... while a pool that always fits finishes in the first launch, so the relaunch takes fewer pools
    assert any(max(n) <= cap for n in need)


# ------------------------------------------------------------------------------------------ tiers
def test_pools_per_launch_at_every_tier_edge(sms):
    c4, c3, c2 = pool_capacity(sms, 4), pool_capacity(sms, 3), pool_capacity(sms, 2)
    assert c4 < c3 < c2
    with tsb200.NQueensEvaluator(17, M=c2 + 1) as ev:
        for M, want in ((1, 4), (c4, 4), (c4 + 1, 3), (c3, 3), (c3 + 1, 2), (c2, 2), (c2 + 1, 1)):
            assert ev.pools_per_launch(M) == want, M


# ------------------------------------------------------------------------------------------ whole searches
def search_counts(golden_dir, N):
    if N <= 3:
        r = po.nq_search_seq(N)
        return r.tree, r.sol
    if N == 18:
        h = json.load(open(os.path.join(golden_dir, "nqueens_depth_hist.json")))["18"]
        return sum(h.values()), h["18"]
    c = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    return c["tree"], c["sol"]


@pytest.mark.parametrize("N", list(range(1, 19)))
def test_whole_search_default_configuration(golden_dir, N, monkeypatch):
    """M = 50 000, m = 25, several pools per task and stealing (the bench's configuration)"""
    monkeypatch.delenv("TSB200_POOLS", raising=False)
    monkeypatch.delenv("TSB200_NO_STEAL", raising=False)
    want = search_counts(golden_dir, N)
    if N == 18:
        assert want == (59365844490, 666090624)
    st = tsb200.nqueens_search_device(N, 1, 25, 50000, 1)
    assert (st.explored_tree, st.explored_sol) == want
    with tsb200.NQueensEvaluator(N, M=50000) as ev:
        st = ev.search(25, 50000)
    assert (st.explored_tree, st.explored_sol) == want


def test_whole_search_n17_big_chunks(golden_dir, monkeypatch):
    """M = 2^22: two-kernel rounds (pool_step), the bench's nqueens_N17_bigM leg"""
    monkeypatch.delenv("TSB200_POOLS", raising=False)
    monkeypatch.delenv("TSB200_NO_STEAL", raising=False)
    with tsb200.NQueensEvaluator(17, M=1 << 22) as ev:
        st = ev.search(25, 1 << 22)
    assert (st.explored_tree, st.explored_sol) == search_counts(golden_dir, 17)

"""The persistent PFSP kernel (csrc/pfsp_rounds.cuh, tsb_pfsp_pool_run for lb1 / lb1_d) against the oracle's pool
loop (po.pfsp_expand applied round by round to a host pool), not against another path of this library: at every edge
of its grid and of its sub-slice split, on every machine count and value-range route of pfsp_shapes.npz, with
IMPROVED exits from rounds whose slices span two tiles, at the incumbent's ties and int32 clamps, with roots in the
chunk, and over whole searches whose incumbent falls.

Every size that depends on the GPU is derived at run time from tsb_device_sm_count with the formulas of
pfsp_rounds_grid (csrc/tsb200_api.cu) and of the kernel's sub-slice split, so the file holds on any SM count.  Every
edge test asserts that it reached its edge: the chunk of the round, the grid, the tiles a slice spans, slow_rounds
(the rounds a leaf improved, which leave the kernel and are redone by tsb_pfsp_pool_step) and kernel launches."""
import json
import os
import zlib

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po
from test_gpu_pfsp_shapes import open_handle
from test_oracle import SHAPE_TAGS, SHAPES

pytestmark = pytest.mark.gpu

PF_TILE, PFR_TILES, PFR_MAX_CTAS, PFR_MAX_M = 128, 3, 256, 20000  # pfsp_kernels.cuh, pfsp_rounds.cuh
PFR_SLICE = PFR_TILES * PF_TILE
JOBS = 20
OPT = {14: 1377, 21: 2297}
INT_MAX = 2**31 - 1
INT64_MAX = 2**63 - 1
NODE = tsb200.PFSP_NODE_DTYPE


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


@pytest.fixture(autouse=True)
def default_routes(monkeypatch):
    """no environment switch of the library leaks in from the caller's environment"""
    for v in ("TSB200_NO_SIMD16", "TSB200_NO_ROUNDS", "TSB200_POOL_CAP"):
        monkeypatch.delenv(v, raising=False)


@pytest.fixture(scope="module")
def sms():
    n = int(tsb200.lib().tsb_device_sm_count(0))
    assert n > 0
    return n


@pytest.fixture(scope="module")
def shapes():
    return np.load(SHAPES)


# ------------------------------------------------------------------------------------------ grid and slices
def rounds_grid(sms, M):
    """pfsp_rounds_grid for lb1 / lb1_d: CTAs of the persistent kernel for chunks of up to M parents; 0: the loop of
    tsb_pfsp_pool_step runs instead"""
    s = min(sms, PFR_MAX_CTAS)
    if M > PFR_MAX_M or M > s * PFR_SLICE:
        return 0
    return min(s, -(-M // PF_TILE))


def sub_slices(n, G):
    """(a0, len0, a1, len1) of each CTA k for a chunk of n parents: sub-slice k from the bottom, k from the top"""
    G2 = 2 * G
    out = []
    for k in range(G):
        a0, a1 = n * k // G2, n * (G2 - 1 - k) // G2
        out.append((a0, n * (k + 1) // G2 - a0, a1, n * (G2 - k) // G2 - a1))
    return out


def tiles_per_slice(n, G):
    """the most 128-parent tiles one CTA's slice spans"""
    return max(-(-(l0 + l1) // PF_TILE) for _, l0, _, l1 in sub_slices(n, G))


# ------------------------------------------------------------------------------------------ nodes
def nodes(rng, count, lo, hi):
    """`count` nodes the search can create: depth lo..hi, limit1 = depth - 1, prmu a permutation of 0..19"""
    out = np.zeros(count, dtype=NODE)
    depth = rng.integers(lo, hi + 1, size=count)
    out["depth"], out["limit1"] = depth, depth - 1
    out["prmu"] = np.argsort(rng.random((count, JOBS)), axis=1).astype(np.int32)
    return out


def roots(rng, count):
    """depth-0 nodes (limit1 = -1): the identity permutation first, then random ones"""
    out = np.zeros(count, dtype=NODE)
    out["limit1"] = -1
    out["prmu"] = np.argsort(rng.random((count, JOBS)), axis=1).astype(np.int32)
    out["prmu"][0] = np.arange(JOBS)
    return out


def ov(a):
    return np.ascontiguousarray(a).view(po.PFSP_NODE_DTYPE)


def live_bounds(t, lb, chunk):
    """the oracle's bounds of the live slots (k >= limit1 + 1) of every node, at best = INT_MAX"""
    b = po.pfsp_evaluate(t, tsb200.LB_NAMES[lb], ov(chunk), INT_MAX).reshape(-1, JOBS)
    return b, po.pfsp_live_mask(ov(chunk), JOBS)


def median_bound(t, lb, rng, lo, hi):
    """an incumbent that keeps about half of the children of depth lo..hi nodes"""
    b, live = live_bounds(t, lb, nodes(rng, 2000, lo, hi))
    return int(np.median(b[live]))


# ------------------------------------------------------------------------------------------ the oracle's pool loop
class OraclePfspPool:
    """The reference's PFSP offload loop on the host: popBackBulk(m, M) -> evaluate + generate_children
    (po.pfsp_expand, the sequential rule: a leaf lowers best while the chunk is walked) -> children appended.  Each
    round is recorded with its chunk size, children, solutions and the incumbent before and after it."""

    def __init__(self, t, lb, start):
        self.t, self.kind = t, tsb200.LB_NAMES[lb]
        self.pool = np.ascontiguousarray(start, dtype=NODE).copy()
        self.rounds = []

    @property
    def size(self):
        return self.pool.shape[0]

    def step(self, m, M, best):
        """one round; None when the pool holds fewer than m nodes"""
        size = self.size
        if size < m:
            return None
        n = min(size, M)
        s0 = size - n
        kids, sol, after = po.pfsp_expand(self.t, self.kind, ov(self.pool[s0:]), best)
        self.pool = np.concatenate([self.pool[:s0], kids.view(NODE)])
        r = dict(parents=n, children=kids.shape[0], solutions=sol, best_in=best, best_out=after)
        self.rounds.append(r)
        return r

    def run(self, m, M, best, max_rounds):
        """tsb_pfsp_pool_run: ([rounds, parents, children, solutions], best after)"""
        tot = [0, 0, 0, 0]
        while tot[0] < max_rounds:
            r = self.step(m, M, best)
            if r is None:
                break
            best = r["best_out"]
            tot = [tot[0] + 1, tot[1] + r["parents"], tot[2] + r["children"], tot[3] + r["solutions"]]
        return tot, best


def improved(r):
    return r["best_out"] < r["best_in"]


def run_and_check(ev, o, lb, m, M, best, max_rounds):
    """one pool_run call against the oracle's loop: counters, incumbent, pool size, and slow_rounds: exactly the
    rounds in which a leaf lowered the incumbent leave the kernel (IMPROVED) and are redone by pool_step"""
    slow0, r0 = ev.slow_rounds, len(o.rounds)
    got = ev.pool_run(lb, m, M, best, max_rounds=max_rounds)
    want, wbest = o.run(m, M, best, max_rounds)
    assert list(got[:4]) == want and got[4] == wbest, (M, max_rounds, got, want, wbest)
    assert ev.pool_size == o.size
    assert ev.slow_rounds - slow0 == sum(improved(r) for r in o.rounds[r0:])
    return wbest


def assert_pool(ev, o, push_back=True):
    """the device pool holds the oracle's pool byte for byte (pushed back afterwards: the next launch starts from a
    freshly pushed arena)"""
    assert ev.pool_size == o.size
    got = ev.pool_drain()
    assert ev.pool_size == 0
    assert got.tobytes() == o.pool.tobytes()
    if push_back and got.shape[0]:
        ev.pool_push(got)


def run_calls(ev, o, lb, m, M, best, calls):
    """pool_run in calls of `calls` rounds: each call resumes from the stack the previous launch left"""
    for k in calls:
        best = run_and_check(ev, o, lb, m, M, best, k)
    return best


def first_round_in_kernel(ev, o, lb, m, M, best):
    """pool_run(max_rounds=1) whose round stays in the persistent kernel: one launch, no slow round"""
    launches = ev.kernel_launches
    best = run_and_check(ev, o, lb, m, M, best, 1)
    assert not improved(o.rounds[-1])
    assert ev.kernel_launches == launches + 1
    return best


# ------------------------------------------------------------------------------------------ grid edges
def edge_Ms(sms):
    S = min(sms, PFR_MAX_CTAS)
    Ms = {1, 2, 127, 128, 129, 256, 257, PF_TILE * S - 1, PF_TILE * S, PF_TILE * S + 1, 20000}
    return sorted(M for M in Ms if M <= min(PFR_MAX_M, PFR_SLICE * S))


@pytest.mark.parametrize("scalar", [False, True], ids=["simd16", "scalar"])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
@pytest.mark.parametrize("inst", [14, 21])
def test_grid_edges(inst, lb, scalar, sms, monkeypatch):
    """G = 1 (M <= 128), M = 1, m = 1; one tile per CTA at M = 128 G_max and two at 128 G_max + 1; first chunks of
    n = 1, 2G - 1, 2G, 2G + 1 and M parents; and a pool that crosses M between two rounds of one launch"""
    if scalar:
        monkeypatch.setenv("TSB200_NO_SIMD16", "1")
    t = po.tables(inst, heads_mode=0)
    rng = np.random.default_rng(9100 + 10 * inst + 2 * (lb == "lb1") + scalar)
    # depth 4..17: no leaf in the first round (it stays in the kernel); leaves and IMPROVED exits come later
    best = median_bound(t, lb, rng, 4, 17)
    S = min(sms, PFR_MAX_CTAS)
    seen = {"G1": False, "one_tile_full": False, "two_tiles": False, "empty_sub_slices": False, "unequal": False,
            "crossing": False}
    with tsb200.PfspEvaluator(inst, M=PFR_MAX_M) as ev:
        if scalar:
            assert not ev.route & tsb200.ROUTE_SIMD16
        for M in edge_Ms(sms):
            G = rounds_grid(sms, M)
            assert G > 0
            seen["G1"] |= G == 1
            ns = sorted({n for n in (1, 2 * G - 1, 2 * G, 2 * G + 1, M) if 1 <= n <= M})
            for i, n in enumerate(ns):
                m = 1 if n < 25 or i % 2 else 25
                # a chunk of exactly n: the whole pool when n < M, the top M of a larger pool when n = M
                start = nodes(rng, n if n < M else M + 37, 4, 17)
                o = OraclePfspPool(t, lb, start)
                ev.pool_push(start)
                b = first_round_in_kernel(ev, o, lb, m, M, best)
                assert o.rounds[0]["parents"] == n
                lens = [x for s in sub_slices(n, G) for x in (s[1], s[3])]
                seen["empty_sub_slices"] |= 0 in lens
                seen["unequal"] |= n >= 2 * G and min(lens) < max(lens)
                tiles = tiles_per_slice(n, G)
                seen["one_tile_full"] |= G == S and n == PF_TILE * S and tiles == 1
                seen["two_tiles"] |= tiles == 2 and n > PF_TILE * S
                assert_pool(ev, o)
                run_calls(ev, o, lb, m, M, b, (2, 3))
                assert_pool(ev, o, push_back=False)
            if M >= 4:  # the pool crosses M inside one launch: a chunk of M // 2, then (with its children) of M
                start = nodes(rng, M // 2, 2, 6)
                o = OraclePfspPool(t, lb, start)
                ev.pool_push(start)
                launches = ev.kernel_launches
                b = run_and_check(ev, o, lb, 1, M, best, 2)
                assert [r["parents"] for r in o.rounds] == [M // 2, M]
                assert ev.kernel_launches == launches + 1  # both rounds in one launch
                seen["crossing"] = True
                assert_pool(ev, o)
                run_calls(ev, o, lb, 25, M, b, (1, 3))
                assert_pool(ev, o, push_back=False)
    want_two = PF_TILE * S + 1 <= PFR_MAX_M
    assert seen == {**seen, "G1": True, "one_tile_full": True, "empty_sub_slices": True, "unequal": True,
                    "crossing": True, "two_tiles": want_two}


# ------------------------------------------------------------------------------------------ machine counts
J20_TAGS = [t for t in SHAPE_TAGS if t.startswith("j20_")]


def shape_start(rng):
    """a pool like test_expand_and_device_pool's (depth 2..6) with three roots among its nodes"""
    start = nodes(rng, 40, 2, 6)
    r = roots(rng, 3)
    return np.concatenate([r[:1], start[:20], r[1:2], start[20:], r[2:]])


@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
@pytest.mark.parametrize("tag", J20_TAGS)
def test_every_machine_count_and_route(shapes, tag, lb):
    """every 20-job instance of pfsp_shapes.npz (1-20 machines zero-padded to the 5 / 10 / 20 templates, the scalar
    route forced by values, rising min_tails, the lb2-refused ones) at M = 300, with no incumbent (IMPROVED exits)
    and with the median bound of the fixture"""
    rng = np.random.default_rng(zlib.crc32(f"{tag}/{lb}".encode()))
    start = shape_start(rng)
    mid = int(np.median(shapes[f"{tag}_lb1"]))
    ev, t = open_handle(shapes, tag, M=300)
    with ev:
        assert ev.route == int(shapes[f"{tag}_route"][0])
        for best in (INT64_MAX, mid):
            o = OraclePfspPool(t, lb, start)
            ev.pool_push(start)
            b = run_calls(ev, o, lb, 25, 300, best, (1, 2, 37))
            if best == INT64_MAX:
                assert b < INT64_MAX and any(improved(r) for r in o.rounds)  # the pool reached leaves
            assert_pool(ev, o, push_back=False)


@pytest.mark.parametrize("scalar", [False, True], ids=["simd16", "scalar"])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
@pytest.mark.parametrize("tag", ["j20_tl_m04", "j20_tl_m07", "j20_tl_m13"])
def test_machine_templates_at_M_20000(shapes, tag, lb, scalar, sms, monkeypatch):
    """one instance per template (5, 10, 20 machines) at M = 20 000: the pool grows until rounds take more than 128
    parents per CTA (two tiles)"""
    if scalar:
        monkeypatch.setenv("TSB200_NO_SIMD16", "1")
    S = min(sms, PFR_MAX_CTAS)
    if PF_TILE * S + 1 > PFR_MAX_M:
        pytest.skip(f"{S} CTAs take 20 000 parents in one tile each")
    rng = np.random.default_rng(zlib.crc32(f"{tag}/{lb}/{scalar}".encode()))
    start = shape_start(rng)
    ev, t = open_handle(shapes, tag, M=PFR_MAX_M)
    with ev:
        if scalar:
            assert not ev.route & tsb200.ROUTE_SIMD16
        o = OraclePfspPool(t, lb, start)
        ev.pool_push(start)
        run_calls(ev, o, lb, 25, PFR_MAX_M, INT64_MAX, (1, 2, 4))
        assert_pool(ev, o, push_back=False)
    big = [r for r in o.rounds if r["parents"] > PF_TILE * S]
    assert big and any(not improved(r) for r in big)
    assert tiles_per_slice(big[0]["parents"], rounds_grid(sms, PFR_MAX_M)) >= 2


# ------------------------------------------------------------------------------------------ IMPROVED, two tiles
@pytest.mark.parametrize("when", ["first", "later"])
@pytest.mark.parametrize("best", ["max", "loose"])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_improved_exit_from_two_tile_slices(lb, best, when, sms):
    """chunks of 20 000 parents (two tiles per CTA) whose leaves lower the incumbent: in the launch's first round
    (depth-19 parents on top) or in its second (depth-18 parents, whose depth-19 children come next)"""
    S = min(sms, PFR_MAX_CTAS)
    if PF_TILE * S + 1 > PFR_MAX_M:
        pytest.skip(f"{S} CTAs take 20 000 parents in one tile each")
    M = PFR_MAX_M
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9300 + 4 * (lb == "lb1") + 2 * (best == "max") + (when == "first"))
    top = nodes(rng, M - 3000, 18, 19) if when == "first" else nodes(rng, M - 3000, 17, 18)
    start = np.concatenate([nodes(rng, M, 8, 12), top])
    b0 = INT64_MAX if best == "max" else 5000
    o = OraclePfspPool(t, lb, start)
    with tsb200.PfspEvaluator(14, M=M) as ev:
        ev.pool_push(start)
        slow0 = ev.slow_rounds
        run_calls(ev, o, lb, 25, M, b0, (1, 2, 3))
        assert ev.slow_rounds > slow0
        assert_pool(ev, o, push_back=False)
    first = next(i for i, r in enumerate(o.rounds) if improved(r))
    assert first == (0 if when == "first" else 1)
    assert o.rounds[first]["parents"] > PF_TILE * S
    assert tiles_per_slice(o.rounds[first]["parents"], rounds_grid(sms, M)) >= 2


# ------------------------------------------------------------------------------------------ ties and clamps
@pytest.mark.parametrize("scalar", [False, True], ids=["simd16", "scalar"])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_leaf_tie_stays_in_the_kernel(lb, scalar, monkeypatch):
    """a chunk of depth-19 parents whose smallest leaf bound is L: with best = L no leaf improves (the round is the
    kernel's: one launch, no slow round); with best = L + 1 one round leaves the kernel and best becomes L"""
    if scalar:
        monkeypatch.setenv("TSB200_NO_SIMD16", "1")
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9400 + 2 * (lb == "lb1") + scalar)
    below = nodes(rng, 300, 8, 12)  # (no leaf within the rounds below)
    chunk = nodes(rng, 500, 19, 19)
    b, _ = live_bounds(t, lb, chunk)
    L = int(b[:, 19].min())
    assert (b[:, 19] == L).sum() >= 1
    start = np.concatenate([below, chunk])
    for best, slow in ((L, 0), (L + 1, 1)):
        o = OraclePfspPool(t, lb, start)
        with tsb200.PfspEvaluator(14, M=500) as ev:
            ev.pool_push(start)
            launches = ev.kernel_launches
            got = run_and_check(ev, o, lb, 1, 500, best, 1)
            assert got == L and o.rounds[0]["parents"] == 500 and o.rounds[0]["solutions"] == 500
            assert ev.slow_rounds == slow
            if slow == 0:
                assert ev.kernel_launches == launches + 1
            assert_pool(ev, o)
            run_calls(ev, o, lb, 1, 500, got, (2, 3))
            assert_pool(ev, o, push_back=False)
            assert ev.slow_rounds == slow


@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_child_tie_is_pruned(lb):
    """best = B, a bound some non-leaf child has, with B <= every leaf bound: the children with bound B are pruned,
    the ones below B pushed, and the round stays in the kernel"""
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9500 + (lb == "lb1"))
    start = np.concatenate([nodes(rng, 200, 19, 19), nodes(rng, 300, 8, 14)])
    b, live = live_bounds(t, lb, start)
    deep = start["depth"] == 19
    L = int(b[deep, 19].min())
    inner = b[~deep][live[~deep]]
    cand = np.unique(inner[inner <= L])
    B = int(cand[cand.size // 2])
    assert B <= L and (inner == B).sum() > 0 and (inner < B).sum() > 0
    o = OraclePfspPool(t, lb, start)
    with tsb200.PfspEvaluator(14, M=500) as ev:
        ev.pool_push(start)
        best = first_round_in_kernel(ev, o, lb, 1, 500, B)
        assert best == B and o.rounds[0]["children"] == (inner < B).sum()
        assert_pool(ev, o)
        run_calls(ev, o, lb, 1, 500, best, (2, 3))
        assert_pool(ev, o, push_back=False)


@pytest.mark.parametrize("best", [2**31 - 1, 2**31, 2**40, 2**63 - 1, 0, -1, -2**40])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_incumbent_clamping(lb, best):
    """incumbents beyond the int32 range are clamped for the kernel and keep the oracle's int64 semantics: at or
    above INT32_MAX nothing is pruned and the first leaves lower best; at or below 0 nothing survives"""
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9600 + (lb == "lb1"))
    start = np.concatenate([nodes(rng, 400, 2, 19), roots(rng, 2)])
    o = OraclePfspPool(t, lb, start)
    with tsb200.PfspEvaluator(14, M=300) as ev:
        ev.pool_push(start)
        after = run_calls(ev, o, lb, 1, 300, best, (1, 2, 5))
        assert_pool(ev, o, push_back=False)
    if best <= 0:
        assert all(r["children"] == 0 for r in o.rounds) and after == best
    else:
        assert any(improved(r) for r in o.rounds) and after < INT_MAX


# ------------------------------------------------------------------------------------------ roots
@pytest.mark.parametrize("M", [64, 300])
@pytest.mark.parametrize("lb", ["lb1_d", "lb1"])
def test_roots_among_deeper_nodes(lb, M):
    """depth-0 parents (limit1 = -1; lb1_d starts from min_heads) mixed with deeper nodes, m = 1"""
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9700 + M + (lb == "lb1"))
    start = np.concatenate([roots(rng, 10), nodes(rng, 60, 3, 15)])[rng.permutation(70)]
    start = np.concatenate([start, roots(rng, 1)])  # (the identity root on top: in the first chunk)
    assert (start[-M:]["depth"] == 0).sum() >= 2
    o = OraclePfspPool(t, lb, start)
    with tsb200.PfspEvaluator(14, M=M) as ev:
        ev.pool_push(start)
        best = first_round_in_kernel(ev, o, lb, 1, M, OPT[14])
        assert_pool(ev, o)
        run_calls(ev, o, lb, 1, M, best, (2, 5))
        assert_pool(ev, o, push_back=False)


@pytest.mark.parametrize("k", [54, 55, 100])
@pytest.mark.parametrize("lb", ["lb1_d", "lb1"])
def test_first_round_of_roots_exactly_fills_the_arena(lb, k, monkeypatch):
    """k roots in an arena of 20 k records (TSB200_POOL_CAP): the first round's worst case, k parents with 20
    children each, fills it exactly (it runs in the kernel); the next round's does not fit (SPACE exit, growth)"""
    cap = JOBS * k
    assert cap >= k + 1024  # (the first push allocates max(TSB200_POOL_CAP, k + 1024) records)
    monkeypatch.setenv("TSB200_POOL_CAP", str(cap))
    t = po.tables(14, heads_mode=0)
    rng = np.random.default_rng(9800 + k + (lb == "lb1"))
    start = roots(rng, k)
    o = OraclePfspPool(t, lb, start)
    M = 300
    with tsb200.PfspEvaluator(14, M=M) as ev:
        ev.pool_push(start)
        best = first_round_in_kernel(ev, o, lb, 1, M, OPT[14])
        assert o.rounds[0]["parents"] * JOBS == cap
        run_and_check(ev, o, lb, 1, M, best, 6)
        assert_pool(ev, o, push_back=False)
    size1 = o.rounds[0]["children"]
    n1 = min(size1, M)
    assert size1 - n1 + n1 * JOBS > cap  # the second round had to grow the arena


@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_pool_run_from_the_root_to_exhaustion(golden_dir, lb):
    """the ta014 root, m = 1, M = 20 000, best = the optimum: the whole tree in pool_run calls (the twin of the
    N-Queens test_pool_run_to_exhaustion_counts); the oracle's loop gives the reference's counts"""
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["pfsp"]
    want = counts["ta014_lb1_ub1" if lb == "lb1" else "ta014_lb0_ub1"]
    root = roots(np.random.default_rng(0), 1)
    with tsb200.PfspEvaluator(14, M=PFR_MAX_M) as ev:
        ev.pool_push(root)
        got = ev.pool_run(lb, 1, PFR_MAX_M, OPT[14])
        assert (got[2], got[3], got[4]) == (want["tree"], want["sol"], want["best"])
        assert ev.pool_size == 0 and ev.slow_rounds == 0
        assert ev.kernel_launches < got[0]


# ------------------------------------------------------------------------------------------ whole searches
# po.pfsp_search_offload(14, lb, 0, 25, M, 1): (tree, solutions, best, offloads, offloaded parents).  The oracle
# takes 10 - 46 s per search on one CPU core, so its values are kept here.
SEARCHES = {("lb1_d", 300): (41016172, 1112952, 1377, 136726, 41016144),
            ("lb1_d", 6000): (42464284, 1131686, 1377, 7085, 42464267),
            ("lb1", 20000): (46055445, 1172484, 1377, 2313, 46055441)}


@pytest.mark.parametrize("lb,M", list(SEARCHES))
def test_whole_search_with_a_falling_incumbent(lb, M, monkeypatch):
    """ub = 0 (best starts at the int64 maximum): leaves keep lowering best, so the offload loop alternates between
    the persistent kernel, IMPROVED exits, pool_step rounds and relaunches"""
    monkeypatch.setenv("TSB200_NO_STEAL", "1")
    st = tsb200.pfsp_search_device(14, lb, 0, 25, M, 1)
    got = (st.explored_tree, st.explored_sol, st.best, st.offloads, st.offloaded_parents)
    assert got == SEARCHES[(lb, M)]
    assert st.kernel_launches < st.offloads

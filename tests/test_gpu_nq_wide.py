"""Wide N-Queens handles (tsb_nq_create_wide: a MAX_QUEENS = 24 build, 25-byte nodes) on the GPU (`pytest -m gpu`):
evaluate and expand against the oracle built with OR_MAX_QUEENS = 24 for N = 1..24 at the chunk edges and on every host
route; the device pool's step / run / drain / steal against the oracle's pool loop on N = 21..24 subtrees, byte for
byte after every round; whole searches with N <= 20 on the wide route against the narrow handle's counts, and
N = 21..24 subtree searches against the reference's counts (tests/golden/nqueens_wide.json)."""
import json
import os

import numpy as np
import pytest

import tsb200
from oracle import pyoracle24 as po24
from test_gpu_host_routes import M_MAX, PIPE_CHUNK, Problem, route_matrix

pytestmark = pytest.mark.gpu
W = tsb200.NQ_NODE24_DTYPE
EDGES = (1, 127, 128, 129, 511, 512, 513)


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


def rand_nodes(rng, N, count, depth_lo=0):
    nodes = np.zeros(count, dtype=W)
    nodes["depth"] = rng.integers(min(depth_lo, N), N + 1, size=count)
    nodes["board"][:, :N] = np.argsort(rng.random((count, N)), axis=1).astype(np.uint8)
    return nodes


def live_mask(parents, N):
    return np.arange(N)[None, :] >= parents["depth"][:, None].astype(np.int64)


def subtree_root(N, prefix):
    node = np.zeros(1, dtype=W)
    b = node["board"][0]
    b[:N] = np.arange(N)
    for d, col in enumerate(prefix):
        j = int(np.nonzero(b[:N] == col)[0][0])
        b[d], b[j] = b[j], b[d]
    node["depth"] = len(prefix)
    return node


def goldens(golden_dir):
    return json.load(open(os.path.join(golden_dir, "nqueens_wide.json")))["subtrees"]


# ------------------------------------------------------------------------------------------ evaluate
@pytest.mark.parametrize("kernel", ["small", "tma"])
@pytest.mark.parametrize("N", range(1, 25))
def test_evaluate_at_the_chunk_edges(N, kernel, monkeypatch):
    if kernel == "tma":
        monkeypatch.setenv("TSB200_NQ_TILE_THREADS", "128")  # the TMA-pipelined kernel at every chunk size
    M = 1500
    parents = rand_nodes(np.random.default_rng(N), N, M)
    want = po24.nq_evaluate(parents, N).reshape(M, N)
    live = live_mask(parents, N)
    with tsb200.NQueensEvaluator(N, M=M, max_queens=24) as ev:
        assert ev.wide and ev.node_dtype == W
        assert len(ev.evaluate(parents[:0])) == 0
        for count in EDGES + (M,):
            got = ev.evaluate(parents[:count]).reshape(count, N)
            assert np.array_equal(np.where(live[:count], got, 0), np.where(live[:count], want[:count], 0)), count


@pytest.mark.parametrize("N", [21, 24])
def test_evaluate_large_chunk_takes_the_tma_kernel(N):
    M = 140000  # more than two 512-parent tiles per SM of an H100
    parents = rand_nodes(np.random.default_rng(50 + N), N, M)
    with tsb200.NQueensEvaluator(N, M=M) as ev:
        got = ev.evaluate(parents).reshape(M, N)
    live = live_mask(parents, N)
    assert np.array_equal(np.where(live, got, 0), np.where(live, po24.nq_evaluate(parents, N).reshape(M, N), 0))


@pytest.mark.parametrize("kernel", ["small", "tma"])
@pytest.mark.parametrize("N", [1, 13, 20, 21, 24])
def test_evaluate_routes(N, kernel, monkeypatch):
    """every registration x alignment x transfer mode x count (tests/test_gpu_host_routes.py's matrix)"""
    monkeypatch.setenv("TSB200_PIPE_MIN", "1")
    monkeypatch.setenv("TSB200_PIPE_CHUNK", str(PIPE_CHUNK))
    if kernel == "tma":
        monkeypatch.setenv("TSB200_NQ_TILE_THREADS", "128")
    parents = rand_nodes(np.random.default_rng(300 + N), N, M_MAX)
    with tsb200.NQueensEvaluator(N, M=M_MAX, max_queens=24) as ev:
        call = lambda p, n, o: tsb200.lib().tsb_nq_evaluate(ev._h, p, n, o)  # noqa: E731
        pb = Problem(ev, parents, N, np.uint8, call, po24.nq_evaluate(parents, N).reshape(M_MAX, N),
                     live_mask(parents, N))
        route_matrix(pb, 128 if kernel == "small" else 512)


def test_evaluate_device_on_a_caller_stream():
    import torch
    N, M = 22, 3000
    parents = rand_nodes(np.random.default_rng(7), N, M)
    with tsb200.NQueensEvaluator(N, M=16) as ev:  # (count is not limited by M_max on the device form)
        d_in = torch.from_numpy(parents.view(np.uint8).copy()).cuda()
        d_out = torch.zeros(M * N, dtype=torch.uint8, device="cuda")
        s = torch.cuda.Stream()
        ev.evaluate_device(d_in.data_ptr(), M, d_out.data_ptr(), s.cuda_stream)
        s.synchronize()
        got = d_out.cpu().numpy().reshape(M, N)
    live = live_mask(parents, N)
    assert np.array_equal(np.where(live, got, 0), np.where(live, po24.nq_evaluate(parents, N).reshape(M, N), 0))


# ------------------------------------------------------------------------------------------ expand
@pytest.mark.parametrize("N", range(1, 25))
def test_expand_at_the_chunk_edges(N):
    M = 1500
    parents = rand_nodes(np.random.default_rng(100 + N), N, M, depth_lo=max(0, N - 6))
    with tsb200.NQueensEvaluator(N, M=M, max_queens=24) as ev:
        kids, sol = ev.expand(parents[:0])
        assert len(kids) == 0 and sol == 0
        for count in EDGES + (M,):
            kids, sol = ev.expand(np.ascontiguousarray(parents[:count]))
            wk, ws = po24.nq_expand(np.ascontiguousarray(parents[:count]), N)
            assert sol == ws and kids.tobytes() == wk.tobytes(), count


@pytest.mark.parametrize("N", [20, 21, 24])
def test_expand_device_dense_tiles_and_unaligned_children(N):
    """shallow parents have up to N - depth children each: dense tiles (several item windows); the children are
    written at an odd byte offset"""
    import torch
    M = 5000
    parents = rand_nodes(np.random.default_rng(200 + N), N, M)
    parents["depth"] = np.random.default_rng(1).integers(0, 4, size=M)
    wk, ws = po24.nq_expand(parents, N)
    with tsb200.NQueensEvaluator(N, M=M, max_queens=24) as ev:
        d_in = torch.from_numpy(parents.view(np.uint8).copy()).cuda()
        d_out = torch.full((M * N * 25 + 64,), 0xEE, dtype=torch.uint8, device="cuda")
        nc, ns = ev.expand_device(d_in.data_ptr(), M, d_out.data_ptr() + 3)
        out = d_out.cpu().numpy()
    assert (nc, ns) == (wk.shape[0], ws)
    assert out[3:3 + 25 * nc].tobytes() == wk.tobytes()
    assert (out[:3] == 0xEE).all() and (out[3 + 25 * nc:] == 0xEE).all()


# ------------------------------------------------------------------------------------------ device pool
class ModelPool:
    """the reference's Pool of one task with the oracle's offload rounds (popBackBulk(m, M), evaluate_gpu,
    generate_children)"""

    def __init__(self, N):
        self.N, self.pool = N, np.zeros(0, dtype=W)

    def push(self, nodes):
        self.pool = np.concatenate([self.pool, nodes])

    def step(self, m, M):
        if self.pool.shape[0] < m:
            return 0, 0, 0
        n = min(self.pool.shape[0], M)
        s0 = self.pool.shape[0] - n
        kids, sol = po24.nq_expand(np.ascontiguousarray(self.pool[s0:]), self.N)
        self.pool = np.concatenate([self.pool[:s0], kids])
        return n, kids.shape[0], sol

    def steal_to(self, thief, m):
        if self.pool.shape[0] < 2 * m:
            return 0
        k = self.pool.shape[0] // 2
        thief.push(self.pool[:k])
        self.pool = self.pool[k:].copy()
        return k


def check_pool(ev, model, tag):
    """the device pool's logical content equals the model's (drained, compared, pushed back)"""
    got = ev.pool_drain()
    assert got.tobytes() == model.pool.tobytes(), tag
    ev.pool_push(got)


@pytest.mark.parametrize("N", [21, 22, 23, 24])
def test_pool_rounds_match_the_oracle_loop(N, golden_dir, monkeypatch):
    monkeypatch.setenv("TSB200_POOL_CAP", "4096")  # small arenas: the rounds compact and grow them
    s = [x for x in goldens(golden_dir) if x["N"] == N][-1]
    root = subtree_root(N, s["prefix"])
    m, M = 5, 3000
    with tsb200.NQueensEvaluator(N, M=M) as ev, tsb200.NQueensEvaluator(N, M=M) as thief:
        assert ev.wide and ev.pools_per_launch(M) == 1
        model, tmodel = ModelPool(N), ModelPool(N)
        ev.pool_push(root)
        model.push(root)
        for r in range(12):
            assert ev.pool_step(m, M) == model.step(m, M), r
            check_pool(ev, model, f"round {r}")
        assert thief.pool_steal_from(ev, m) == model.steal_to(tmodel, m)
        check_pool(ev, model, "victim after the steal")
        check_pool(thief, tmodel, "thief after the steal")
        for _ in range(3):  # pool_run is the pool_step loop: compare it with the model's rounds
            want = [0, 0, 0, 0]
            for _ in range(7):
                n, c, so = model.step(m, M)
                if n == 0:
                    break
                want = [want[0] + 1, want[1] + n, want[2] + c, want[3] + so]
            assert list(ev.pool_run(m, M, max_rounds=7)) == want
            check_pool(ev, model, "after pool_run")
        assert ev.pool_size == model.pool.shape[0] and thief.pool_size == tmodel.pool.shape[0]


def test_pool_push_admits_only_nodes_the_search_can_create():
    N = 21
    with tsb200.NQueensEvaluator(N, M=100) as ev:
        good = subtree_root(N, [0, 2, 4])
        ev.pool_push(good)
        for mutate in (lambda x: x.__setitem__("depth", N + 1),
                       lambda x: x["board"].__setitem__((0, N), 1),  # a byte past N
                       lambda x: x["board"].__setitem__((0, 23), 1),
                       lambda x: x["board"].__setitem__((0, 3), N)):
            bad = good.copy()
            mutate(bad)
            with pytest.raises(tsb200.TsbError) as e:
                ev.pool_push(bad)
            assert e.value.code == tsb200._lib.EINVAL
        assert ev.pool_size == 1 and ev.pool_drain().tobytes() == good.tobytes()


def test_steal_and_shared_runs_take_wide_handles_only_together():
    with tsb200.NQueensEvaluator(14, M=100) as narrow, tsb200.NQueensEvaluator(14, M=100, max_queens=24) as wide:
        for a, b in ((narrow, wide), (wide, narrow)):
            with pytest.raises(tsb200.TsbError) as e:
                a.pool_steal_from(b, 1)
            assert e.value.code == tsb200._lib.EINVAL
            with pytest.raises(tsb200.TsbError) as e:
                tsb200.nqueens_pool_run_multi([a, b], 1, 100)
            assert e.value.code == tsb200._lib.EINVAL
        assert tsb200.lib().tsb_nq_max_queens(wide._h) == 24 and tsb200.lib().tsb_nq_max_queens(narrow._h) == 20


def test_pool_run_multi_runs_wide_pools_one_after_the_other(golden_dir):
    """two wide pools in one call: each ends where pool_run alone leaves it"""
    N = 21
    roots = [subtree_root(N, s["prefix"]) for s in goldens(golden_dir) if s["N"] == N]
    M = 50000
    evs = [tsb200.NQueensEvaluator(N, M=M) for _ in range(4)]
    try:
        for i, r in enumerate(roots):
            evs[i].pool_push(r)
            evs[2 + i].pool_push(r)
        got = tsb200.nqueens_pool_run_multi(evs[:2], 1, M, max_rounds=40)
        want = [evs[2 + i].pool_run(1, M, max_rounds=40) for i in range(2)]
        assert [tuple(x) for x in got] == [tuple(x) for x in want]
        for i in range(2):
            assert evs[i].pool_drain().tobytes() == evs[2 + i].pool_drain().tobytes()
    finally:
        for ev in evs:
            ev.close()


@pytest.mark.parametrize("s", range(8))
def test_subtree_searches_match_the_reference(s, golden_dir):
    """the device pool from a subtree's root until it is empty: the reference's explored tree and solutions"""
    g = goldens(golden_dir)[s]
    N, M = g["N"], 50000
    with tsb200.NQueensEvaluator(N, M=M) as ev:
        ev.pool_push(subtree_root(N, g["prefix"]))
        rounds, parents, children, sols = ev.pool_run(1, M)
        assert ev.pool_size == 0 and (children, sols) == (g["tree"], g["sol"]) and parents == g["tree"] + 1


# ------------------------------------------------------------------------------------------ whole searches
@pytest.mark.parametrize("D", [1, 2, 3, 4])
@pytest.mark.parametrize("N", [11, 13])
def test_wide_route_searches_equal_the_narrow_counts(N, D, golden_dir):
    """N <= 20 as a MAX_QUEENS = 24 build runs it; D > 1 wraps the tasks onto the GPUs present"""
    want = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    for st in (tsb200.nqueens_search(N, M=2000, D=D, max_queens=24),
               tsb200.nqueens_search_device(N, M=2000, D=D, max_queens=24),
               tsb200.nqueens_search_device(N, M=50000, D=D, max_queens=24)):
        assert (st.explored_tree, st.explored_sol) == (want["tree"], want["sol"])
        assert sum(st.per_gpu_tree[:D]) > 0


@pytest.mark.parametrize("N", [12, 14])
def test_search_on_a_wide_handle(N, golden_dir):
    want = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    with tsb200.NQueensEvaluator(N, M=50000, max_queens=24) as ev:
        st = ev.search(25, 50000)
        launches = ev.kernel_launches
    assert (st.explored_tree, st.explored_sol) == (want["tree"], want["sol"]) and launches > 0

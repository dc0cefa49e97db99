"""CPU checks of the MAX_QUEENS = 24 build (boards of 21 to 24 queens, 25-byte nodes): the oracle built with
OR_MAX_QUEENS = 24 against the reference's own C sources built with MAX_QUEENS 24 (evaluate and decompose), the oracle
against the committed subtree goldens (tests/golden/nqueens_wide.json), and the argument checks of
tsb_nq_create_wide and of the searches, which return before any device is touched."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import tsb200
from oracle import pyoracle24 as po24
from tsb200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
need_ref = pytest.mark.skipif(not po24.ref_available(), reason="oracle/_ref/libref_nqueens24.so is not built")


def rand_nodes(rng, N, count, depth_lo=0):
    """nodes the search can create: a permutation of 0..N-1 on board[0..N), zeros past N, depth in depth_lo..N"""
    nodes = np.zeros(count, dtype=po24.NQ_NODE_DTYPE)
    nodes["depth"] = rng.integers(min(depth_lo, N), N + 1, size=count)
    nodes["board"][:, :N] = np.argsort(rng.random((count, N)), axis=1).astype(np.uint8)
    return nodes


def wide_goldens(golden_dir):
    return json.load(open(os.path.join(golden_dir, "nqueens_wide.json")))


def subtree_root(N, prefix):
    """the node decompose creates for the queens of `prefix` on rows 0, 1, ... (tests/golden/make_golden_nq_wide.py)"""
    node = np.zeros(1, dtype=po24.NQ_NODE_DTYPE)
    b = node["board"][0]
    b[:N] = np.arange(N)
    for d, col in enumerate(prefix):
        j = int(np.nonzero(b[:N] == col)[0][0])
        b[d], b[j] = b[j], b[d]
    node["depth"] = len(prefix)
    return node


# ------------------------------------------------------------------ oracle vs the reference's MAX_QUEENS 24 build
@need_ref
@pytest.mark.parametrize("N", range(1, 25))
def test_evaluate_matches_the_reference_build(N):
    rng = np.random.default_rng(1000 + N)
    parents = rand_nodes(rng, N, 3000)
    assert (po24.nq_evaluate(parents, N) == po24.nq_evaluate(parents, N, use_ref=True)).all()


@need_ref
@pytest.mark.parametrize("N", range(1, 25))
def test_decompose_matches_the_reference_build(N):
    """breadth-first frontiers (decompose's children in order) and searches from random deep nodes"""
    depth = min(N, 3)
    got, gt, gs = po24.nq_frontier(N, depth)
    want, wt, ws = po24.nq_frontier(N, depth, use_ref=True)
    assert (gt, gs) == (wt, ws) and got.shape == want.shape
    # (the reference's decompose copies board[0..N) only: the bytes past N of its children are not defined)
    assert (got["depth"] == want["depth"]).all() and (got["board"][:, :N] == want["board"][:, :N]).all()
    assert not got["board"][:, N:].any()
    rng = np.random.default_rng(2000 + N)
    nodes = rand_nodes(rng, N, 20, depth_lo=max(0, N - 9))
    assert po24.nq_search_from(N, nodes) == po24.nq_search_from(N, nodes, use_ref=True)


# ------------------------------------------------------------------ committed goldens
def test_golden_subtrees_are_reproduced_by_the_oracle(golden_dir):
    g = wide_goldens(golden_dir)
    assert sorted({s["N"] for s in g["subtrees"]}) == [21, 22, 23, 24]
    for s in g["subtrees"]:
        node = subtree_root(s["N"], s["prefix"])
        assert po24.nq_search_from(s["N"], node) == (s["tree"], s["sol"]), s


def test_golden_totals_are_the_published_counts(golden_dir):
    assert wide_goldens(golden_dir)["solutions_oeis_a000170"] == {
        "21": 314666222712, "22": 2691008701644, "23": 24233937684440, "24": 227514171973736}


# ------------------------------------------------------------------ the library's host side
def test_node_layouts():
    assert tsb200.NQ_NODE24_DTYPE.itemsize == 25 and po24.NQ_NODE_DTYPE == tsb200.NQ_NODE24_DTYPE
    assert tsb200.nq_node_dtype(20) == tsb200.NQ_NODE_DTYPE and tsb200.nq_node_dtype(21) == tsb200.NQ_NODE24_DTYPE


@pytest.mark.parametrize("max_queens,N,g,M", [(20, 14, 1, 10), (25, 14, 1, 10), (0, 21, 1, 10), (-24, 21, 1, 10),
                                              (24, 25, 1, 10), (24, 0, 1, 10), (24, -1, 1, 10), (24, 21, 0, 10),
                                              (24, 21, 1, 0)])
def test_create_wide_refuses_bad_arguments(max_queens, N, g, M):
    h = C.c_void_p()
    assert tsb200.lib().tsb_nq_create_wide(C.byref(h), 0, max_queens, N, g, M) == _lib.EINVAL
    assert not h.value


def test_create_wide_refuses_a_null_out_pointer():
    assert tsb200.lib().tsb_nq_create_wide(None, 0, 24, 21, 1, 10) == _lib.EINVAL


def test_narrow_create_still_stops_at_20():
    h = C.c_void_p()
    assert tsb200.lib().tsb_nq_create(C.byref(h), 0, 21, 1, 10) == _lib.EINVAL
    assert tsb200.lib().tsb_nq_max_queens(None) == _lib.EINVAL


def test_searches_refuse_boards_beyond_24():
    L, st = tsb200.lib(), _lib.SearchStats()
    for fn in (L.tsb_nq_search, L.tsb_nq_search_device):
        assert fn(25, 1, 25, 50000, 1, C.byref(st)) == _lib.EINVAL
    assert L.tsb_nq_search_device_part(25, 1, 25, 50000, 1, 0, 0, C.byref(st)) == _lib.EINVAL
    for fn in (L.tsb_nq_search_wide, L.tsb_nq_search_device_wide):
        assert fn(24, 25, 1, 25, 50000, 1, C.byref(st)) == _lib.EINVAL
        assert fn(20, 14, 1, 25, 50000, 1, C.byref(st)) == _lib.EINVAL  # only a MAX_QUEENS = 24 build
    n, t, s = C.c_int64(0), C.c_uint64(0), C.c_uint64(0)
    assert L.tsb_nq_warmup(25, 25, None, 0, C.byref(n), C.byref(t), C.byref(s)) == _lib.EINVAL


@pytest.mark.parametrize("N", [21, 24])
def test_warmup_of_a_wide_board_is_the_reference_breadth_first_pool(N):
    """step 1 (popFront + decompose until the pool holds min_size nodes) with 25-byte nodes"""
    got, tree, sol = tsb200.nqueens_warmup(N, 500)
    assert got.dtype == tsb200.NQ_NODE24_DTYPE
    pool = subtree_root(N, [])
    want_tree = 0
    while pool.shape[0] < 500:
        kids, _ = po24.nq_expand(np.ascontiguousarray(pool[:1]), N)
        pool = np.concatenate([pool[1:], kids])
        want_tree += kids.shape[0]
    assert got.tobytes() == pool.tobytes() and (tree, sol) == (want_tree, 0)


def test_driver_refuses_25_queens():
    exe = os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200", "drivers", "nqueens_b200.out")
    r = subprocess.run([exe, "--N", "25"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 2 and "at most 24 queens" in r.stderr and "Size of the explored tree" not in r.stdout

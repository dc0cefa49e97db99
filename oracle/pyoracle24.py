"""ctypes binding of oracle/liboracle24.so: the CPU oracle (tsb_oracle.c) built with OR_MAX_QUEENS = 24, i.e. the
Chapel program as `chpl -sMAX_QUEENS=24` would build it (lib/nqueens/NQueens_node.chpl:7): 25-byte nodes, N <= 24;
and of oracle/_ref/libref_nqueens24.so, the reference's own C sources built with MAX_QUEENS 24.  Both are built by
oracle/queens24.mk (build()).
TEST INFRASTRUCTURE ONLY, like everything under oracle/."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import pyoracle as po

MAX_QUEENS = 24
NQ_NODE_DTYPE = np.dtype([("depth", np.uint8), ("board", np.uint8, (MAX_QUEENS,))])
assert NQ_NODE_DTYPE.itemsize == 25

_lib = None
_ref = None


def build(ref: bool = True) -> None:
    """compile liboracle24.so (always) and oracle/_ref/libref_nqueens24.so (where the reference checkout exists)"""
    mk = ["make", "-s", "-C", po.HERE, "-f", "queens24.mk"]
    subprocess.run(mk + ["liboracle24.so"], check=True)
    if ref and os.path.isdir(os.path.join(po.REFERENCE, "baselines")):
        subprocess.run(mk + ["ref", f"REF={os.path.abspath(po.REFERENCE)}"], check=True)


_vp, _i32, _u64p = C.c_void_p, C.c_int, C.POINTER(C.c_uint64)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        path = os.path.join(po.HERE, "liboracle24.so")
        if not os.path.exists(path):
            build(ref=False)
        L = C.CDLL(path)
        L.or_nq_evaluate.argtypes = [_vp, _i32, _i32, _i32, _vp]
        L.or_nq_expand_chunk.argtypes = [_vp, _i32, _i32, _i32, _vp, C.c_int64, _u64p]
        L.or_nq_expand_chunk.restype = C.c_int64
        L.or_nq_search_from.argtypes = [_i32, _i32, _vp, _i32, _u64p, _u64p]
        L.or_nq_frontier.argtypes = [_i32, _i32, _i32, _vp, _i32, _u64p, _u64p]
        _lib = L
    return _lib


def ref_path() -> str:
    return os.path.join(po.HERE, "_ref", "libref_nqueens24.so")


def ref_available() -> bool:
    return os.path.exists(ref_path())


def ref() -> C.CDLL:
    """the reference's isSafe / decompose / Pool built with MAX_QUEENS 24 (with oracle/ref_batch.c around them)"""
    global _ref
    if _ref is None:
        L = C.CDLL(ref_path())
        L.ref_nq_evaluate_range.argtypes = [_vp, _i32, _i32, _i32, _i32, _vp]
        L.ref_nq_search_from.argtypes = [_i32, _i32, _vp, _i32, _u64p, _u64p]
        L.ref_nq_frontier.argtypes = [_i32, _i32, _i32, _vp, _i32, _u64p, _u64p]
        _ref = L
    return _ref


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def nq_evaluate(parents: np.ndarray, N: int, g: int = 1, fill: int = 0xCD, use_ref: bool = False) -> np.ndarray:
    """labels[p*N + k] for k >= depth (slots below depth keep `fill`)"""
    assert parents.dtype == NQ_NODE_DTYPE and parents.flags.c_contiguous
    labels = np.full(parents.shape[0] * N, fill, dtype=np.uint8)
    if use_ref:
        ref().ref_nq_evaluate_range(_ptr(parents), 0, parents.shape[0], N, g, _ptr(labels))
    else:
        lib().or_nq_evaluate(_ptr(parents), parents.shape[0], N, g, _ptr(labels))
    return labels


def nq_expand(parents: np.ndarray, N: int, g: int = 1):
    """(children in the reference's order, solutions) of one chunk: evaluate_gpu + generate_children"""
    assert parents.dtype == NQ_NODE_DTYPE and parents.flags.c_contiguous
    cap = max(parents.shape[0] * N, 1)
    out = np.zeros(cap, dtype=NQ_NODE_DTYPE)
    sol = C.c_uint64(0)
    n = lib().or_nq_expand_chunk(_ptr(parents), parents.shape[0], N, g, _ptr(out), cap, C.byref(sol))
    assert 0 <= n <= cap
    return out[:n].copy(), int(sol.value)


def nq_search_from(N: int, nodes: np.ndarray, g: int = 1, use_ref: bool = False):
    """(tree, solutions) of the sequential search (popBack + decompose) started from `nodes`"""
    assert nodes.dtype == NQ_NODE_DTYPE and nodes.flags.c_contiguous
    tree, sol = C.c_uint64(0), C.c_uint64(0)
    fn = ref().ref_nq_search_from if use_ref else lib().or_nq_search_from
    fn(N, g, _ptr(nodes), nodes.shape[0], C.byref(tree), C.byref(sol))
    return int(tree.value), int(sol.value)


def nq_frontier(N: int, depth: int, cap: int = 1 << 20, g: int = 1, use_ref: bool = False):
    """(all nodes of depth `depth`, breadth first from the root, tree, solutions explored on the way)"""
    out = np.zeros(cap, dtype=NQ_NODE_DTYPE)
    tree, sol = C.c_uint64(0), C.c_uint64(0)
    fn = ref().ref_nq_frontier if use_ref else lib().or_nq_frontier
    n = fn(N, g, depth, _ptr(out), cap, C.byref(tree), C.byref(sol))
    assert n >= 0, "frontier larger than cap"
    return out[:n].copy(), int(tree.value), int(sol.value)

"""N-Queens side of the offload interface (nqueens_gpu_chpl.chpl / nqueens_multigpu_chpl.chpl)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import MAX_QUEENS, MAX_QUEENS_WIDE, Evaluator, SearchStats, check, check_search, ckpt_args, lib

# lib/nqueens/NQueens_node.chpl:9-11
NQ_NODE_DTYPE = np.dtype([("depth", np.uint8), ("board", np.uint8, (MAX_QUEENS,))])
assert NQ_NODE_DTYPE.itemsize == 21
# the same record of a build of the reference with MAX_QUEENS = 24 (boards of 21 to 24 queens)
NQ_NODE24_DTYPE = np.dtype([("depth", np.uint8), ("board", np.uint8, (MAX_QUEENS_WIDE,))])
assert NQ_NODE24_DTYPE.itemsize == 25


def nq_node_dtype(N: int) -> np.dtype:
    """the node record of the searches for N queens: 21 bytes up to N = 20, else 25 bytes"""
    return NQ_NODE_DTYPE if N <= MAX_QUEENS else NQ_NODE24_DTYPE


class NQueensEvaluator(Evaluator):
    """Owns what `on device var parents_d, labels_d` owns in the reference (nqueens_gpu_chpl.chpl:194-195).
    N > 20, or max_queens=24 for any N, creates a MAX_QUEENS = 24 handle (tsb_nq_create_wide): its nodes are
    NQ_NODE24_DTYPE records (`node_dtype`), and its device pools run one pool per launch of the persistent kernel."""

    wide, node_dtype = False, NQ_NODE_DTYPE  # (an object that wraps a tsb_nq_create handle)
    _abi = "tsb_nq"

    def __init__(self, N: int, g: int = 1, M: int = 50000, device: int = 0, max_queens: int | None = None):
        self.N, self.g, self.M, self.device = N, g, M, device
        self._h = C.c_void_p()
        if max_queens is None:
            max_queens = MAX_QUEENS if N <= MAX_QUEENS else MAX_QUEENS_WIDE
        self.wide = max_queens != MAX_QUEENS
        self.node_dtype = NQ_NODE24_DTYPE if self.wide else NQ_NODE_DTYPE
        if self.wide:
            check(lib().tsb_nq_create_wide(C.byref(self._h), device, max_queens, N, g, M), "tsb_nq_create_wide")
        else:
            check(lib().tsb_nq_create(C.byref(self._h), device, N, g, M), "tsb_nq_create")

    def evaluate_gpu(self, parents: np.ndarray, size: int, labels: np.ndarray) -> None:
        """evaluate_gpu(parents_d, size, labels_d) of nqueens_gpu_chpl.chpl:97-123 including the copies of
        :203/:205; `size` = N * poolSize as in the reference call (:201-204)."""
        assert parents.dtype == self.node_dtype and parents.flags.c_contiguous
        assert labels.dtype == np.uint8 and labels.flags.c_contiguous
        if size % self.N:
            raise ValueError("size must be N * poolSize")
        count = size // self.N
        assert parents.shape[0] >= count and labels.size >= size
        check(lib().tsb_nq_evaluate(self._h, parents.ctypes.data, count, labels.ctypes.data), "tsb_nq_evaluate")

    def evaluate(self, parents: np.ndarray) -> np.ndarray:
        labels = np.empty(parents.shape[0] * self.N, dtype=np.uint8)
        self.evaluate_gpu(parents, parents.shape[0] * self.N, labels)
        return labels

    # ---- beyond the drop-in: fused evaluate_gpu + generate_children, device-resident pool
    def expand(self, parents: np.ndarray):
        """children of the chunk (packed, reference order) and the number of depth == N parents:
        evaluate_gpu (nqueens_gpu_chpl.chpl:97-123) + generate_children (:126-149) in one device pass"""
        assert parents.dtype == self.node_dtype and parents.flags.c_contiguous
        cap = parents.shape[0] * self.N
        out = np.empty(max(cap, 1), dtype=self.node_dtype)
        nc, ns = C.c_uint64(0), C.c_uint64(0)
        check(lib().tsb_nq_expand(self._h, parents.ctypes.data, parents.shape[0], out.ctypes.data, cap,
                                  C.byref(nc), C.byref(ns)), "tsb_nq_expand")
        return out[: nc.value].copy(), int(ns.value)

    def expand_device(self, parents_ptr: int, count: int, children_ptr: int, stream: int = 0):
        nc, ns = C.c_uint64(0), C.c_uint64(0)
        check(lib().tsb_nq_expand_device(self._h, parents_ptr, count, children_ptr, C.byref(nc), C.byref(ns), stream),
              "tsb_nq_expand_device")
        return int(nc.value), int(ns.value)

    def pool_push(self, nodes: np.ndarray) -> None:
        assert nodes.dtype == self.node_dtype and nodes.flags.c_contiguous
        check(lib().tsb_nq_pool_push(self._h, nodes.ctypes.data, nodes.shape[0]), "tsb_nq_pool_push")

    def pool_step(self, m: int, M: int):
        """(parents popped, children appended, solutions) of one device-side offload round"""
        np_, nc, ns = C.c_int64(0), C.c_uint64(0), C.c_uint64(0)
        check(lib().tsb_nq_pool_step(self._h, m, M, C.byref(np_), C.byref(nc), C.byref(ns)), "tsb_nq_pool_step")
        return int(np_.value), int(nc.value), int(ns.value)

    def search(self, m: int = 25, M: int | None = None) -> SearchStats:
        """the whole 3-step search (nqueens_gpu_chpl.chpl:152-248) with the pool of step 2 on this handle's device"""
        st = SearchStats()
        check(lib().tsb_nq_search_on(self._h, self.N, m, self.M if M is None else M, C.byref(st)), "tsb_nq_search_on")
        return st

    def pools_per_launch(self, M: int) -> int:
        """pools one launch of the persistent kernel serves best for chunks of M parents (tsb_nq_pools_per_launch)"""
        return int(lib().tsb_nq_pools_per_launch(self._h, M))

    def pool_run(self, m: int, M: int, max_rounds: int = 2**62):
        """(rounds, parents popped, children appended, solutions) of up to max_rounds device-side offload rounds
        (until the pool holds fewer than m nodes); one persistent kernel for M <= 512 x #SMs"""
        nr, np_, nc, ns = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        check(lib().tsb_nq_pool_run(self._h, m, M, max_rounds, C.byref(nr), C.byref(np_), C.byref(nc), C.byref(ns)),
              "tsb_nq_pool_run")
        return int(nr.value), int(np_.value), int(nc.value), int(ns.value)

    def evaluate_device(self, parents_ptr: int, count: int, labels_ptr: int, stream: int = 0) -> None:
        """device-resident form; pointers are raw device addresses (e.g. torch.Tensor.data_ptr())"""
        check(lib().tsb_nq_evaluate_device(self._h, parents_ptr, count, labels_ptr, stream), "tsb_nq_evaluate_device")


def nqueens_pool_run_multi(evaluators, m: int, M: int, max_rounds: int = 2**62):
    """up to max_rounds rounds of each evaluator's device pool in shared launches of the persistent kernel
    (tsb_nq_pool_run_multi): [(rounds, parents, children, solutions)] per pool"""
    K = len(evaluators)
    hs = (C.c_void_p * K)(*[ev._h for ev in evaluators])
    out = (C.c_uint64 * (4 * K))()
    check(lib().tsb_nq_pool_run_multi(hs, K, m, M, max_rounds, out), "tsb_nq_pool_run_multi")
    return [tuple(int(out[4 * i + j]) for j in range(4)) for i in range(K)]


def nqueens_warmup(N: int, min_size: int = 25):
    """step 1 of the drivers (nqueens_gpu_chpl.chpl:169-175): (pool nodes, explored tree, solutions); the nodes are
    nq_node_dtype(N) records"""
    cap = max(1024, 32 * min_size)
    out = np.zeros(cap, dtype=nq_node_dtype(N))
    n, tree, sol = C.c_int64(0), C.c_uint64(0), C.c_uint64(0)
    check(lib().tsb_nq_warmup(N, min_size, out.ctypes.data, cap, C.byref(n), C.byref(tree), C.byref(sol)), "tsb_nq_warmup")
    return out[: n.value].copy(), int(tree.value), int(sol.value)


def nqueens_search(N: int = 14, g: int = 1, m: int = 25, M: int = 50000, D: int = 1,
                   max_queens: int | None = None, checkpoint=None, time_limit: float | None = None) -> SearchStats:
    """the 3-step search of nqueens_gpu_chpl.chpl:152-248 (D = 1) / nqueens_multigpu_chpl.chpl:158-352
    (static split, D GPUs), run by the C++ emulation driver inside libtsb200.so.  N in 1..24 (N > 20 with 25-byte
    nodes); max_queens=24: every N as a MAX_QUEENS = 24 build runs it (tsb_nq_search_wide).  checkpoint /
    time_limit: the resumable search (tsb_nq_search_ckpt), as for nqueens_search_device"""
    st = SearchStats()
    if checkpoint is not None:
        mq = MAX_QUEENS if max_queens is None else max_queens
        check_search(lib().tsb_nq_search_ckpt(mq, N, g, m, M, D, *ckpt_args(checkpoint, time_limit), C.byref(st)),
                     "tsb_nq_search_ckpt", st)
    elif max_queens is None:
        check(lib().tsb_nq_search(N, g, m, M, D, C.byref(st)), "tsb_nq_search")
    else:
        check(lib().tsb_nq_search_wide(max_queens, N, g, m, M, D, C.byref(st)), "tsb_nq_search_wide")
    return st


def nqueens_search_device(N: int = 14, g: int = 1, m: int = 25, M: int = 50000, D: int = 1,
                          max_queens: int | None = None, checkpoint=None, time_limit: float | None = None) -> SearchStats:
    """same 3-step search, the pool(s) of step 2 resident on the device(s) (tsb_nq_pool_*).
    checkpoint=path: the resumable search (tsb_nq_search_device_ckpt): it continues from the file if there is one,
    stops after time_limit seconds (None: no limit) or on request_stop() by writing the file and raising
    SearchStopped, and removes the file when it ends; the returned stats are those of the whole search"""
    st = SearchStats()
    if checkpoint is not None:
        mq = MAX_QUEENS if max_queens is None else max_queens
        check_search(lib().tsb_nq_search_device_ckpt(mq, N, g, m, M, D, *ckpt_args(checkpoint, time_limit), C.byref(st)),
                     "tsb_nq_search_device_ckpt", st)
    elif max_queens is None:
        check(lib().tsb_nq_search_device(N, g, m, M, D, C.byref(st)), "tsb_nq_search_device")
    else:
        check(lib().tsb_nq_search_device_wide(max_queens, N, g, m, M, D, C.byref(st)), "tsb_nq_search_device_wide")
    return st


def nqueens_search_device_part(N: int, g: int, m: int, M: int, D: int, part: int, device: int = 0) -> SearchStats:
    """task `part` of the D-way static split on `device` (one rank of a process-per-GPU launch); the parts'
    counts add up to the whole search's"""
    st = SearchStats()
    check(lib().tsb_nq_search_device_part(N, g, m, M, D, part, device, C.byref(st)), "tsb_nq_search_device_part")
    return st

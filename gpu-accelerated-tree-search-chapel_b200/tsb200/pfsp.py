"""PFSP side of the offload interface (pfsp_gpu_chpl.chpl / pfsp_multigpu_chpl.chpl)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import LB1, LB1_D, LB2, Evaluator, PfspTables, PfspTables50, SearchStats, check, check_search, ckpt_args, lib

# lib/pfsp/PFSP_node.chpl:9-12
PFSP_NODE_DTYPE = np.dtype([("depth", np.int32), ("limit1", np.int32), ("prmu", np.int32, (20,))])
assert PFSP_NODE_DTYPE.itemsize == 88
# a build of the reference with MAX_JOBS = 50 (ta031..ta060)
PFSP_NODE50_DTYPE = np.dtype([("depth", np.int32), ("limit1", np.int32), ("prmu", np.int32, (50,))])
assert PFSP_NODE50_DTYPE.itemsize == 208
# the Chapel CLI spells the bounds as strings (pfsp_gpu_chpl.chpl:15), the C ABI as the C baseline's ints
LB_NAMES = {"lb1_d": LB1_D, "lb1": LB1, "lb2": LB2}


def _lb(lb) -> int:
    """the C ABI's code of a bound given as "lb1" | "lb1_d" | "lb2" or as the code itself"""
    return LB_NAMES[lb] if isinstance(lb, str) else int(lb)


LB2_VARIANTS = {"full": 0, "nabeshima": 1, "lageweg": 2, "learn": 3}  # lib/pfsp/Bound_johnson.chpl:6


def taillard_tables(inst: int, variant="full") -> PfspTables:
    """lbound1 / lbound2 as built at pfsp_gpu_chpl.chpl:325-332 (Chapel semantics, incl. its min_heads); `variant`
    selects the machine pairs of lb2 (the reference compiles "full")"""
    t = PfspTables()
    v = LB2_VARIANTS[variant] if isinstance(variant, str) else int(variant)
    check(lib().tsb_pfsp_tables_build_variant(C.byref(t), inst, v), "tsb_pfsp_tables_build_variant")
    return t


def taillard_tables50(inst: int, variant="full") -> PfspTables50:
    t = PfspTables50()
    v = LB2_VARIANTS[variant] if isinstance(variant, str) else int(variant)
    check(lib().tsb_pfsp_tables50_build(C.byref(t), inst, v), "tsb_pfsp_tables50_build")
    return t


class PfspEvaluator(Evaluator):
    """Owns parents_d / bounds_d / lbound1_d / lbound2_d of pfsp_gpu_chpl.chpl:359-371.  Instances with more than
    20 jobs (ta031..ta060) create a MAX_JOBS = 50 handle: nodes are PFSP_NODE50_DTYPE, evaluate only."""

    _abi = "tsb_pfsp"
    pool_dtype = PFSP_NODE_DTYPE  # (the device pool exists for 20 jobs only)

    def __init__(self, inst: int | None = None, tables=None, M: int = 50000, device: int = 0):
        if tables is None:
            tables = taillard_tables50(inst) if lib().tsb_taillard_nb_jobs(inst) > 20 else taillard_tables(inst)
        self.tables = tables
        self.jobs, self.machines, self.M = self.tables.jobs, self.tables.machines, M
        self.wide = isinstance(tables, PfspTables50)
        self.node_dtype = PFSP_NODE50_DTYPE if self.wide else PFSP_NODE_DTYPE
        self._h = C.c_void_p()
        if self.wide:
            check(lib().tsb_pfsp_create50_from_tables(C.byref(self._h), device, M, C.byref(self.tables)), "tsb_pfsp_create_wide")
        else:
            check(lib().tsb_pfsp_create_from_tables(C.byref(self._h), device, M, C.byref(self.tables)), "tsb_pfsp_create")

    def evaluate_gpu(self, parents: np.ndarray, size: int, best: int, lb, bounds: np.ndarray) -> None:
        """evaluate_gpu(parents_d, size, best, lbound1_d, lbound2_d, bounds_d) of pfsp_gpu_chpl.chpl:257-270 with
        the copies of :384/:386; `size` = jobs * poolSize; lb is "lb1" | "lb1_d" | "lb2" or the int code"""
        assert parents.dtype == self.node_dtype and parents.flags.c_contiguous
        assert bounds.dtype == np.int32 and bounds.flags.c_contiguous
        kind = _lb(lb)
        if size % self.jobs:
            raise ValueError("size must be jobs * poolSize")
        count = size // self.jobs
        assert parents.shape[0] >= count and bounds.size >= size
        check(lib().tsb_pfsp_evaluate(self._h, kind, parents.ctypes.data, count, int(best), bounds.ctypes.data),
              "tsb_pfsp_evaluate")

    def evaluate(self, parents: np.ndarray, lb, best: int) -> np.ndarray:
        bounds = np.empty(parents.shape[0] * self.jobs, dtype=np.int32)
        self.evaluate_gpu(parents, parents.shape[0] * self.jobs, best, lb, bounds)
        return bounds

    def evaluate_device(self, lb, parents_ptr: int, count: int, best: int, bounds_ptr: int, stream: int = 0) -> None:
        kind = _lb(lb)
        check(lib().tsb_pfsp_evaluate_device(self._h, kind, parents_ptr, count, int(best), bounds_ptr, stream),
              "tsb_pfsp_evaluate_device")


    # ---- beyond the drop-in: fused evaluate_gpu + generate_children, device-resident pool
    def expand(self, parents: np.ndarray, lb, best: int):
        """(children, n_solutions, best_after): evaluate_gpu (pfsp_gpu_chpl.chpl:192-270) + generate_children
        (:273-303) of one chunk in one device pass"""
        assert parents.dtype == PFSP_NODE_DTYPE and parents.flags.c_contiguous
        kind = _lb(lb)
        cap = parents.shape[0] * self.jobs
        out = np.empty(max(cap, 1), dtype=PFSP_NODE_DTYPE)
        nc, ns, b = C.c_uint64(0), C.c_uint64(0), C.c_int64(int(best))
        check(lib().tsb_pfsp_expand(self._h, kind, parents.ctypes.data, parents.shape[0], C.byref(b), out.ctypes.data,
                                    cap, C.byref(nc), C.byref(ns)), "tsb_pfsp_expand")
        return out[: nc.value].copy(), int(ns.value), int(b.value)

    def expand_device(self, lb, parents_ptr: int, count: int, best: int, children_ptr: int, stream: int = 0):
        """(n_children, n_solutions, best_after) of expand on device arrays (parents 16-byte aligned, children 8-byte
        aligned), ordered on `stream` (0: the handle's stream)"""
        kind = _lb(lb)
        nc, ns, b = C.c_uint64(0), C.c_uint64(0), C.c_int64(int(best))
        check(lib().tsb_pfsp_expand_device(self._h, kind, parents_ptr, count, C.byref(b), children_ptr, C.byref(nc),
                                           C.byref(ns), stream), "tsb_pfsp_expand_device")
        return int(nc.value), int(ns.value), int(b.value)

    def pool_push(self, nodes: np.ndarray) -> None:
        assert nodes.dtype == PFSP_NODE_DTYPE and nodes.flags.c_contiguous
        check(lib().tsb_pfsp_pool_push(self._h, nodes.ctypes.data, nodes.shape[0]), "tsb_pfsp_pool_push")

    @property
    def slow_rounds(self) -> int:
        return int(lib().tsb_pfsp_slow_rounds(self._h))

    @property
    def route(self) -> int:
        """tsb_pfsp_route: template machine count | ROUTE_SIMD16 | ROUTE_LB2 | ROUTE_LB2U"""
        r = int(lib().tsb_pfsp_route(self._h))
        check(min(r, 0), "tsb_pfsp_route")
        return r

    def pool_step(self, lb, m: int, M: int, best: int):
        """(parents popped, children appended, solutions, best_after) of one device-side offload round"""
        kind = _lb(lb)
        np_, nc, ns, b = C.c_int64(0), C.c_uint64(0), C.c_uint64(0), C.c_int64(int(best))
        check(lib().tsb_pfsp_pool_step(self._h, kind, m, M, C.byref(b), C.byref(np_), C.byref(nc), C.byref(ns)),
              "tsb_pfsp_pool_step")
        return int(np_.value), int(nc.value), int(ns.value), int(b.value)

    def pool_run(self, lb, m: int, M: int, best: int, max_rounds: int = 2**62):
        """(rounds, parents, children, solutions, best_after): pool_step rounds until the pool holds fewer than m
        nodes or max_rounds are done, for lb1 / lb1_d and M up to 20 000 in one persistent kernel"""
        kind = _lb(lb)
        b = C.c_int64(int(best))
        nr, np_, nc, ns = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        check(lib().tsb_pfsp_pool_run(self._h, kind, m, M, max_rounds, C.byref(b), C.byref(nr), C.byref(np_),
                                      C.byref(nc), C.byref(ns)), "tsb_pfsp_pool_run")
        return int(nr.value), int(np_.value), int(nc.value), int(ns.value), int(b.value)

    def search(self, inst: int, lb, ub: int = 1, m: int = 25, M: int | None = None, pools: int = 1) -> SearchStats:
        """the whole 3-step search (pfsp_gpu_chpl.chpl:306-431) with the pool of step 2 on this handle's device;
        pools > 1: on this handle and its first pools - 1 siblings (tsb_pfsp_search_on_pools)"""
        kind = _lb(lb)
        st = SearchStats()
        M = self.M if M is None else M
        if pools == 1:
            check(lib().tsb_pfsp_search_on(self._h, inst, kind, ub, m, M, C.byref(st)), "tsb_pfsp_search_on")
        else:
            check(lib().tsb_pfsp_search_on_pools(self._h, inst, kind, ub, m, M, pools, C.byref(st)),
                  "tsb_pfsp_search_on_pools")
        return st

    def sibling(self, index: int) -> "PfspEvaluator":
        """further device pool `index` (1..3) with this evaluator's tables, device and M (tsb_pfsp_sibling): the
        same evaluator on every call; its handle belongs to this evaluator and is destroyed with it"""
        sibs = self.__dict__.setdefault("_siblings", {})
        h = C.c_void_p()
        check(lib().tsb_pfsp_sibling(self._h, index, C.byref(h)), "tsb_pfsp_sibling")
        if index not in sibs:
            sib = PfspEvaluator.__new__(PfspEvaluator)
            sib.__dict__.update(tables=self.tables, jobs=self.jobs, machines=self.machines, M=self.M, wide=self.wide,
                                node_dtype=self.node_dtype, _h=h, _owner=self)
            sibs[index] = sib
        return sibs[index]

    def pools_per_launch(self, lb, M: int) -> int:
        """pools one launch of the persistent kernel can serve for chunks of M parents (tsb_pfsp_pools_per_launch)"""
        kind = _lb(lb)
        return int(lib().tsb_pfsp_pools_per_launch(self._h, kind, M))



def pfsp_pool_run_multi(evaluators, lb, m: int, M: int, bests, max_rounds: int = 2**62):
    """up to max_rounds rounds of each evaluator's device pool, each with its own incumbent, in shared launches of the
    persistent kernel (tsb_pfsp_pool_run_multi): [(rounds, parents, children, solutions, best_after)] per pool"""
    kind = _lb(lb)
    K = len(evaluators)
    if len(bests) != K:
        raise ValueError("one incumbent per pool")
    hs = (C.c_void_p * K)(*[ev._h for ev in evaluators])
    b = (C.c_int64 * K)(*[int(x) for x in bests])
    out = (C.c_uint64 * (4 * K))()
    check(lib().tsb_pfsp_pool_run_multi(hs, K, kind, m, M, max_rounds, b, out), "tsb_pfsp_pool_run_multi")
    return [tuple(int(out[4 * i + j]) for j in range(4)) + (int(b[i]),) for i in range(K)]


def pfsp_search_device(inst: int = 14, lb="lb1", ub: int = 1, m: int = 25, M: int = 50000, D: int = 1,
                       pools: int = 1, checkpoint=None, time_limit: float | None = None) -> SearchStats:
    """same search, the pool(s) of step 2 resident on the device(s) (tsb_pfsp_pool_*); pools > 1: that many device
    pools per task (tsb_pfsp_search_device_pools).  checkpoint / time_limit: the resumable search
    (tsb_pfsp_search_device_ckpt), as for nqueens_search_device"""
    kind = _lb(lb)
    st = SearchStats()
    if checkpoint is not None:
        check_search(lib().tsb_pfsp_search_device_ckpt(inst, kind, ub, m, M, D, pools, *ckpt_args(checkpoint, time_limit),
                                                       C.byref(st)), "tsb_pfsp_search_device_ckpt", st)
    elif pools == 1:
        check(lib().tsb_pfsp_search_device(inst, kind, ub, m, M, D, C.byref(st)), "tsb_pfsp_search_device")
    else:
        check(lib().tsb_pfsp_search_device_pools(inst, kind, ub, m, M, D, pools, C.byref(st)),
              "tsb_pfsp_search_device_pools")
    return st


def pfsp_search(inst: int = 14, lb="lb1", ub: int = 1, m: int = 25, M: int = 50000, D: int = 1,
                checkpoint=None, time_limit: float | None = None) -> SearchStats:
    """pfsp_gpu_chpl.chpl:306-431 (D = 1) / pfsp_multigpu_chpl.chpl (static split), C++ emulation driver.
    checkpoint / time_limit: the resumable search (tsb_pfsp_search_ckpt), as for nqueens_search_device"""
    kind = _lb(lb)
    st = SearchStats()
    if checkpoint is not None:
        check_search(lib().tsb_pfsp_search_ckpt(inst, kind, ub, m, M, D, *ckpt_args(checkpoint, time_limit),
                                                C.byref(st)), "tsb_pfsp_search_ckpt", st)
    else:
        check(lib().tsb_pfsp_search(inst, kind, ub, m, M, D, C.byref(st)), "tsb_pfsp_search")
    return st


MAX_JOBS_WIDE = 50


def pfsp_search_wide(inst: int = 31, lb="lb1", ub: int = 1, m: int = 25, M: int = 50000, D: int = 1,
                     checkpoint=None, time_limit: float | None = None) -> SearchStats:
    """pfsp_search as the reference built with MAX_JOBS = 50 runs it (tsb_pfsp_search_wide): ta031..ta060, 208-byte
    nodes (with checkpoint / time_limit the resumable tsb_pfsp_search_ckpt_wide)"""
    kind = _lb(lb)
    st = SearchStats()
    if checkpoint is not None:
        check_search(lib().tsb_pfsp_search_ckpt_wide(MAX_JOBS_WIDE, inst, kind, ub, m, M, D,
                                                     *ckpt_args(checkpoint, time_limit), C.byref(st)),
                     "tsb_pfsp_search_ckpt_wide", st)
    else:
        check(lib().tsb_pfsp_search_wide(MAX_JOBS_WIDE, inst, kind, ub, m, M, D, C.byref(st)), "tsb_pfsp_search_wide")
    return st


def pfsp_search_device_wide(inst: int = 31, lb="lb1", ub: int = 1, m: int = 25, M: int = 50000, D: int = 1,
                            pools: int = 1, checkpoint=None, time_limit: float | None = None) -> SearchStats:
    """pfsp_search_device as the reference built with MAX_JOBS = 50 runs it (tsb_pfsp_search_device_wide; with
    checkpoint / time_limit the resumable tsb_pfsp_search_device_ckpt_wide)"""
    kind = _lb(lb)
    st = SearchStats()
    if checkpoint is not None:
        check_search(lib().tsb_pfsp_search_device_ckpt_wide(MAX_JOBS_WIDE, inst, kind, ub, m, M, D, pools,
                                                            *ckpt_args(checkpoint, time_limit), C.byref(st)),
                     "tsb_pfsp_search_device_ckpt_wide", st)
    else:
        check(lib().tsb_pfsp_search_device_wide(MAX_JOBS_WIDE, inst, kind, ub, m, M, D, pools, C.byref(st)),
              "tsb_pfsp_search_device_wide")
    return st


def pfsp_search_device_part(inst: int, lb, ub: int, m: int, M: int, D: int, part: int, device: int = 0,
                            pools: int = 1) -> SearchStats:
    kind = _lb(lb)
    st = SearchStats()
    if pools == 1:
        check(lib().tsb_pfsp_search_device_part(inst, kind, ub, m, M, D, part, device, C.byref(st)),
              "tsb_pfsp_search_device_part")
    else:
        check(lib().tsb_pfsp_search_device_pools_part(inst, kind, ub, m, M, D, pools, part, device, C.byref(st)),
              "tsb_pfsp_search_device_pools_part")
    return st

"""ctypes loader for the CPU ORACLE (oracle/liboracle.so) and, when present, the reference's own
C sources compiled into oracle/_ref/ (see oracle/Makefile).

TEST INFRASTRUCTURE ONLY — imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
# the reference checkout whose C sources `build(ref=True)` compiles into oracle/_ref: $TSB200_REFERENCE, by default a
# directory `reference` next to this repository (oracle/Makefile uses the same default)
REFERENCE = os.environ.get("TSB200_REFERENCE") or os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference")
MAX_JOBS = 20
MAX_MACHINES = 20
MAX_QUEENS = 20

NQ_NODE_DTYPE = np.dtype([("depth", np.uint8), ("board", np.uint8, (MAX_QUEENS,))])  # 21 B
PFSP_NODE_DTYPE = np.dtype([("depth", np.int32), ("limit1", np.int32), ("prmu", np.int32, (MAX_JOBS,))])  # 88 B
assert NQ_NODE_DTYPE.itemsize == 21 and PFSP_NODE_DTYPE.itemsize == 88


class Tables(C.Structure):
    """mirror of or_pfsp_tables (oracle/tsb_oracle.h)"""

    _fields_ = [
        ("jobs", C.c_int32),
        ("machines", C.c_int32),
        ("pairs", C.c_int32),
        ("p_times", C.c_int32 * (MAX_MACHINES * MAX_JOBS)),
        ("min_heads", C.c_int32 * MAX_MACHINES),
        ("min_tails", C.c_int32 * MAX_MACHINES),
        ("johnson", C.c_int32 * (190 * MAX_JOBS)),
        ("lags", C.c_int32 * (190 * MAX_JOBS)),
        ("mp0", C.c_int32 * 190),
        ("mp1", C.c_int32 * 190),
        ("mp_order", C.c_int32 * 190),
    ]

    def arr(self, name, n=None):
        a = np.ctypeslib.as_array(getattr(self, name))
        return a[:n].copy() if n is not None else a.copy()


class SearchResult(C.Structure):
    _fields_ = [
        ("tree", C.c_uint64),
        ("sol", C.c_uint64),
        ("best", C.c_int64),
        ("offloads", C.c_uint64),
        ("offloaded_parents", C.c_uint64),
        ("live_slots", C.c_uint64),
        ("depth_hist", C.c_uint64 * (MAX_JOBS + 2)),
        ("seconds", C.c_double),
        ("task_tree", C.c_uint64 * 8),
        ("task_sol", C.c_uint64 * 8),
        ("task_best", C.c_int64 * 8),
    ]


def build(ref: bool = True) -> None:
    """compile liboracle.so (always) and oracle/_ref (where the reference checkout REFERENCE exists)"""
    subprocess.run(["make", "-s", "-C", HERE, "liboracle.so", "liboracle50.so"], check=True)
    if ref and os.path.isdir(os.path.join(REFERENCE, "baselines")):
        subprocess.run(["make", "-s", "-C", HERE, "ref", f"REF={os.path.abspath(REFERENCE)}"], check=True)


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        path = os.path.join(HERE, "liboracle.so")
        if not os.path.exists(path):
            build(ref=False)
        L = C.CDLL(path)
        vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
        L.or_taillard_nb_jobs.restype = C.c_int32
        L.or_taillard_nb_machines.restype = C.c_int32
        L.or_taillard_best_ub.restype = C.c_int64
        L.or_taillard_processing_times.argtypes = [vp, i32]
        L.or_pfsp_tables_build.argtypes = [C.POINTER(Tables), i32, i32]
        L.or_pfsp_tables_build_variant.argtypes = [C.POINTER(Tables), i32, i32, i32]
        L.or_pfsp_tables_from_ptimes.argtypes = [C.POINTER(Tables), i32, i32, vp, i32, i32]
        L.or_eval_solution.argtypes = [C.POINTER(Tables), vp]
        L.or_eval_solution.restype = C.c_int32
        L.or_lb1_bound.argtypes = [C.POINTER(Tables), vp, C.c_int32, C.c_int32]
        L.or_lb1_bound.restype = C.c_int32
        L.or_lb1_children_bounds.argtypes = [C.POINTER(Tables), vp, C.c_int32, C.c_int32, vp]
        L.or_lb2_bound.argtypes = [C.POINTER(Tables), vp, C.c_int32, C.c_int32, i64]
        L.or_lb2_bound.restype = C.c_int32
        L.or_nq_evaluate.argtypes = [vp, i32, i32, i32, vp]
        L.or_nq_evaluate_range.argtypes = [vp, i32, i32, i32, i32, vp]
        L.or_pfsp_evaluate.argtypes = [C.POINTER(Tables), i32, vp, i32, i64, vp]
        L.or_pfsp_evaluate_range.argtypes = [C.POINTER(Tables), i32, vp, i32, i32, i64, vp]
        L.or_nq_expand_chunk.argtypes = [vp, i32, i32, i32, vp, i64, C.POINTER(C.c_uint64)]
        L.or_nq_expand_chunk.restype = C.c_int64
        L.or_pfsp_expand_chunk.argtypes = [vp, i32, vp, i32, C.POINTER(C.c_int64), vp, i64, C.POINTER(C.c_uint64)]
        L.or_pfsp_expand_chunk.restype = C.c_int64
        L.or_nq_search_seq.argtypes = [i32, i32, C.POINTER(SearchResult)]
        L.or_nq_search_from.argtypes = [i32, i32, vp, i32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.or_nq_frontier.argtypes = [i32, i32, i32, vp, i32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.or_nq_search_offload.argtypes = [i32, i32, i32, i32, i32, C.POINTER(SearchResult)]
        L.or_pfsp_search_seq.argtypes = [i32, i32, i32, i32, C.POINTER(SearchResult)]
        L.or_pfsp_search_offload.argtypes = [i32, i32, i32, i32, i32, i32, i32, C.POINTER(SearchResult)]
        L.or_nq_search_offload_part.argtypes = [i32, i32, i32, i32, i32, i32, i32, C.POINTER(SearchResult)]
        L.or_pfsp_search_offload_part.argtypes = [i32, i32, i32, i32, i32, i32, i32, i32, C.POINTER(SearchResult)]
        L.or_nq_capture_chunk.argtypes = [i32, i32, i32, i32, i32, vp, i32]
        L.or_pfsp_capture_chunk.argtypes = [i32, i32, i32, i32, i32, i32, vp, i32, C.POINTER(C.c_int64)]
        _lib = L
    return _lib


# ---------------------------------------------------------------- convenience wrappers

LB2_VARIANTS = {"full": 0, "nabeshima": 1, "lageweg": 2, "learn": 3}  # lib/pfsp/Bound_johnson.chpl:6


def tables(inst: int, heads_mode: int = 0, variant: int = 0) -> Tables:
    t = Tables()
    rc = lib().or_pfsp_tables_build_variant(C.byref(t), inst, heads_mode, variant)
    if rc != 0:
        raise ValueError(f"or_pfsp_tables_build({inst}) -> {rc}")
    return t


def tables_from_ptimes(p_times, heads_mode: int = 0, variant: int = 0, L=None, cls=Tables):
    """the tables fill_* build from a processing-time matrix p_times[machines, jobs] (any values)"""
    p = np.ascontiguousarray(p_times, dtype=np.int32)
    machines, jobs = p.shape
    t = cls()
    rc = (L or lib()).or_pfsp_tables_from_ptimes(C.byref(t), jobs, machines, _ptr(p), heads_mode, variant)
    if rc != 0:
        raise ValueError(f"or_pfsp_tables_from_ptimes({jobs} jobs, {machines} machines) -> {rc}")
    return t


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def nq_evaluate(parents: np.ndarray, N: int, g: int = 1, fill: int = 0xCD) -> np.ndarray:
    """labels[count*N]; slots the reference does not write keep `fill`"""
    assert parents.dtype == NQ_NODE_DTYPE and parents.flags.c_contiguous
    labels = np.full(parents.shape[0] * N, fill, dtype=np.uint8)
    lib().or_nq_evaluate(_ptr(parents), parents.shape[0], N, g, _ptr(labels))
    return labels


def pfsp_evaluate(t: Tables, lb_kind: int, parents: np.ndarray, best: int, fill: int = -0x32323233) -> np.ndarray:
    assert parents.dtype == PFSP_NODE_DTYPE and parents.flags.c_contiguous
    bounds = np.full(parents.shape[0] * t.jobs, fill, dtype=np.int32)
    lib().or_pfsp_evaluate(C.byref(t), lb_kind, _ptr(parents), parents.shape[0], int(best), _ptr(bounds))
    return bounds


def nq_expand(parents: np.ndarray, N: int, g: int = 1):
    """(children, n_solutions) of one chunk in the reference's generate_children order"""
    assert parents.dtype == NQ_NODE_DTYPE and parents.flags.c_contiguous
    cap = parents.shape[0] * N + 1
    out = np.zeros(cap, dtype=NQ_NODE_DTYPE)
    sol = C.c_uint64(0)
    n = lib().or_nq_expand_chunk(_ptr(parents), parents.shape[0], N, g, _ptr(out), cap, C.byref(sol))
    return out[:n].copy(), int(sol.value)


def pfsp_expand(t: Tables, lb_kind: int, parents: np.ndarray, best: int):
    """(children, n_solutions, best_after) of one chunk: bounds with `best` at launch, then the reference's
    sequential generate_children"""
    assert parents.dtype == PFSP_NODE_DTYPE and parents.flags.c_contiguous
    cap = parents.shape[0] * t.jobs + 1
    out = np.zeros(cap, dtype=PFSP_NODE_DTYPE)
    sol = C.c_uint64(0)
    b = C.c_int64(int(best))
    n = lib().or_pfsp_expand_chunk(C.byref(t), lb_kind, _ptr(parents), parents.shape[0], C.byref(b), _ptr(out), cap,
                                   C.byref(sol))
    return out[:n].copy(), int(sol.value), int(b.value)


def nq_live_mask(parents: np.ndarray, N: int) -> np.ndarray:
    """boolean [count, N]: slots k >= depth (the only slots the contract defines)"""
    return np.arange(N)[None, :] >= parents["depth"][:, None].astype(np.int64)


def pfsp_live_mask(parents: np.ndarray, jobs: int) -> np.ndarray:
    return np.arange(jobs)[None, :] >= (parents["limit1"][:, None].astype(np.int64) + 1)


def nq_search_seq(N, g=1):
    r = SearchResult()
    lib().or_nq_search_seq(N, g, C.byref(r))
    return r


def nq_search_offload(N, g=1, m=25, M=50000, D=1):
    r = SearchResult()
    lib().or_nq_search_offload(N, g, m, M, D, C.byref(r))
    return r


def pfsp_search_seq(inst, lb_kind, ub=1, heads_mode=0):
    r = SearchResult()
    lib().or_pfsp_search_seq(inst, lb_kind, ub, heads_mode, C.byref(r))
    return r


def pfsp_search_offload(inst, lb_kind, ub=1, m=25, M=50000, D=1, heads_mode=0):
    r = SearchResult()
    lib().or_pfsp_search_offload(inst, lb_kind, ub, m, M, D, heads_mode, C.byref(r))
    return r


def _check_part(D, part):
    if not (1 <= D <= 8 and 0 <= part < D):
        raise ValueError(f"part {part} of a {D}-way split")


def nq_search_offload_part(N, g=1, m=25, M=50000, D=1, part=0, warm=None):
    """task `part` of the D-way split run alone (or_nq_search_offload_part); warm: the step-1 pool size, D * m by
    default"""
    _check_part(D, part)
    r = SearchResult()
    lib().or_nq_search_offload_part(N, g, m, M, D, part, D * m if warm is None else warm, C.byref(r))
    return r


def pfsp_search_offload_part(inst, lb_kind, ub=1, m=25, M=50000, D=1, part=0, heads_mode=0):
    _check_part(D, part)
    r = SearchResult()
    lib().or_pfsp_search_offload_part(inst, lb_kind, ub, m, M, D, part, heads_mode, C.byref(r))
    return r


def nq_capture_chunk(N, which, g=1, m=25, M=50000) -> np.ndarray:
    out = np.zeros(M, dtype=NQ_NODE_DTYPE)
    n = lib().or_nq_capture_chunk(N, g, m, M, which, _ptr(out), M)
    if n < 0:
        raise IndexError(f"offload #{which} does not exist for N={N}")
    return out[:n].copy()


def pfsp_capture_chunk(inst, lb_kind, which, ub=1, m=25, M=50000):
    out = np.zeros(M, dtype=PFSP_NODE_DTYPE)
    best = C.c_int64(0)
    n = lib().or_pfsp_capture_chunk(inst, lb_kind, ub, m, M, which, _ptr(out), M, C.byref(best))
    if n < 0:
        raise IndexError(f"offload #{which} does not exist")
    return out[:n].copy(), int(best.value)


# ---------------------------------------------------------------- the reference's own C code (oracle/_ref)

class RefLb1(C.Structure):  # baselines/pfsp/lib/c_bound_simple.h:14-21
    _fields_ = [("p_times", C.POINTER(C.c_int)), ("min_heads", C.POINTER(C.c_int)),
                ("min_tails", C.POINTER(C.c_int)), ("nb_jobs", C.c_int), ("nb_machines", C.c_int)]


class RefLb2(C.Structure):  # baselines/pfsp/lib/c_bound_johnson.h:18-29
    _fields_ = [("johnson_schedules", C.POINTER(C.c_int)), ("lags", C.POINTER(C.c_int)),
                ("machine_pairs_1", C.POINTER(C.c_int)), ("machine_pairs_2", C.POINTER(C.c_int)),
                ("machine_pair_order", C.POINTER(C.c_int)), ("nb_machine_pairs", C.c_int),
                ("nb_jobs", C.c_int), ("nb_machines", C.c_int)]


def ref_available() -> bool:
    return all(os.path.exists(os.path.join(HERE, "_ref", f)) for f in ("libref_nqueens.so", "libref_pfsp.so"))


_ref_nq = None
_ref_pf = None


def ref_nqueens() -> C.CDLL:
    global _ref_nq
    if _ref_nq is None:
        L = C.CDLL(os.path.join(HERE, "_ref", "libref_nqueens.so"))
        # uint8_t isSafe(const int G, const uint8_t* board, const uint8_t queen_num, const uint8_t row_pos)
        L.isSafe.argtypes = [C.c_int, C.c_void_p, C.c_uint8, C.c_uint8]
        L.isSafe.restype = C.c_uint8
        L.ref_nq_evaluate_range.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.ref_nq_evaluate_range_rep.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
        if hasattr(L, "ref_nq_search_from"):  # (an oracle/_ref built before round 2 lacks the search harness)
            L.ref_nq_search_from.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_uint64),
                                             C.POINTER(C.c_uint64)]
            L.ref_nq_frontier.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_uint64),
                                          C.POINTER(C.c_uint64)]
        _ref_nq = L
    return _ref_nq


def nq_cpu_search(N: int, threads: int, depth: int = 3, use_ref: bool | None = None):
    """the reference's sequential N-Queens search (nqueens_c.c:112-141; nqueens_chpl.chpl:92-113) on `threads` host
    threads: the subtrees below the breadth-first frontier of depth `depth` are handed out dynamically, each explored
    with the reference's own pool / isSafe / decompose (oracle/_ref; the oracle port if that is absent).  Returns
    (explored_tree, solutions, seconds, "reference" | "port")"""
    import itertools
    import threading
    import time
    use_ref = ref_available() and hasattr(ref_nqueens(), "ref_nq_search_from") if use_ref is None else use_ref
    L = ref_nqueens() if use_ref else lib()
    frontier_fn = L.ref_nq_frontier if use_ref else L.or_nq_frontier
    search_fn = L.ref_nq_search_from if use_ref else L.or_nq_search_from
    cap = 1 << 16
    nodes = np.zeros(cap, dtype=NQ_NODE_DTYPE)
    tree, sol = C.c_uint64(0), C.c_uint64(0)
    t0 = time.perf_counter()
    n = frontier_fn(N, 1, min(depth, N), _ptr(nodes), cap, C.byref(tree), C.byref(sol))
    assert n >= 0
    ticket = itertools.count()  # (next() on it is atomic under the GIL)
    parts = [[0, 0] for _ in range(threads)]

    def work(w):
        t_, s_ = C.c_uint64(0), C.c_uint64(0)
        base = nodes.ctypes.data
        while True:
            i = next(ticket)
            if i >= n:
                break
            search_fn(N, 1, base + i * NQ_NODE_DTYPE.itemsize, 1, C.byref(t_), C.byref(s_))  # (GIL released)
        parts[w] = [t_.value, s_.value]

    th = [threading.Thread(target=work, args=(w,)) for w in range(threads)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    dt = time.perf_counter() - t0
    return (tree.value + sum(p[0] for p in parts), sol.value + sum(p[1] for p in parts), dt,
            "reference" if use_ref else "port")


_ref_pf_chapel = None


def ref_pfsp(chapel_heads: bool = False) -> C.CDLL:
    """the reference's PFSP C sources as a library; chapel_heads=True: the build in which the one line of
    fill_min_heads_tails that differs from the Chapel program says what the Chapel line says (oracle/Makefile)"""
    global _ref_pf, _ref_pf_chapel
    if chapel_heads:
        if _ref_pf_chapel is None:
            _ref_pf_chapel = _load_ref_pfsp("libref_pfsp_chapel.so")
        return _ref_pf_chapel
    if _ref_pf is None:
        _ref_pf = _load_ref_pfsp("libref_pfsp.so")
    return _ref_pf


def _load_ref_pfsp(name: str) -> C.CDLL:
    if True:
        L = C.CDLL(os.path.join(HERE, "_ref", name))
        L.new_bound_data.argtypes = [C.c_int, C.c_int]
        L.new_bound_data.restype = C.POINTER(RefLb1)
        L.new_johnson_bd_data.argtypes = [C.POINTER(RefLb1)]
        L.new_johnson_bd_data.restype = C.POINTER(RefLb2)
        L.taillard_get_processing_times.argtypes = [C.POINTER(C.c_int), C.c_int]
        L.fill_min_heads_tails.argtypes = [C.POINTER(RefLb1)]
        L.fill_machine_pairs.argtypes = [C.POINTER(RefLb2)]
        L.fill_lags.argtypes = [C.POINTER(C.c_int), C.POINTER(RefLb2)]
        L.fill_johnson_schedules.argtypes = [C.POINTER(C.c_int), C.POINTER(RefLb2)]
        L.lb1_bound.argtypes = [C.POINTER(RefLb1), C.c_void_p, C.c_int, C.c_int]
        L.lb1_bound.restype = C.c_int
        L.lb1_children_bounds.argtypes = [C.POINTER(RefLb1), C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.lb2_bound.argtypes = [C.POINTER(RefLb1), C.POINTER(RefLb2), C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.lb2_bound.restype = C.c_int
        L.eval_solution.argtypes = [C.POINTER(RefLb1), C.c_void_p]
        L.eval_solution.restype = C.c_int
        L.ref_pfsp_evaluate_range.argtypes = [C.POINTER(RefLb1), C.POINTER(RefLb2), C.c_int, C.c_void_p, C.c_int,
                                              C.c_int, C.c_int, C.c_void_p]
        L.ref_pfsp_evaluate_range_rep.argtypes = [C.POINTER(RefLb1), C.POINTER(RefLb2), C.c_int, C.c_void_p, C.c_int,
                                                  C.c_int, C.c_int, C.c_void_p, C.c_int]
    return L


_ref_named = {}


def ref_pfsp_named(name: str) -> C.CDLL:
    """another build of the reference's PFSP sources (oracle/Makefile): "nabeshima" / "lageweg" (lb2 variants),
    "50" (MAX_JOBS = 50)"""
    if name not in _ref_named:
        _ref_named[name] = _load_ref_pfsp(f"libref_pfsp{name if name == '50' else '_' + name}.so")
    return _ref_named[name]


def ref_pfsp_data(inst: int, chapel_heads: bool = False, L=None):
    """(lb1*, lb2*) built by the reference's own functions, as pfsp_c.c:236-246 does"""
    L = L or ref_pfsp(chapel_heads)
    jobs, machines = lib().or_taillard_nb_jobs(inst), lib().or_taillard_nb_machines(inst)
    d1 = L.new_bound_data(jobs, machines)
    L.taillard_get_processing_times(d1.contents.p_times, inst)
    L.fill_min_heads_tails(d1)
    d2 = L.new_johnson_bd_data(d1)
    L.fill_machine_pairs(d2)
    L.fill_lags(d1.contents.p_times, d2)
    L.fill_johnson_schedules(d1.contents.p_times, d2)
    return d1, d2

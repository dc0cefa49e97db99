"""ctypes binding of libtsb200.so (include/tsb200.h).  Fails loudly if the CUDA extension is missing:
there is no CPU fallback anywhere in this package."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

PKG_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.environ.get("TSB200_LIB") or os.path.join(PKG_DIR, "libtsb200.so")  # (TSB200_LIB: A/B builds)

MAX_JOBS = 20
MAX_QUEENS, MAX_QUEENS_WIDE = 20, 24
MAX_MACHINES = 20
MAX_PAIRS = 190

OK, EINVAL, ECUDA, ENOMEM, ENODEV, EALIGN, EUNSUPPORTED, ESTOPPED = 0, -1, -2, -3, -4, -5, -6, -7
LB1_D, LB1, LB2 = 0, 1, 2
XFER_AUTO, XFER_MEMCPY, XFER_ZEROCOPY = 0, 1, 2
# tsb_*_last_xfer: the route of the last host-buffer evaluate call
XFER_ROUTE_ZEROCOPY, XFER_ROUTE_PIPELINED, XFER_ROUTE_IN_STAGED, XFER_ROUTE_OUT_STAGED = 1, 2, 4, 8
# tsb_pfsp_route: template machine count in the low byte, and which kernel specialisations the handle uses
ROUTE_MT_MASK, ROUTE_SIMD16, ROUTE_LB2, ROUTE_LB2U = 0xFF, 0x100, 0x200, 0x400


class TsbError(RuntimeError):
    def __init__(self, code: int, where: str):
        L = lib()
        msg = L.tsb_strerror(code).decode()
        if code == ECUDA:
            msg += " — " + L.tsb_last_cuda_error().decode()
        super().__init__(f"{where}: {msg} ({code})")
        self.code = code


class SearchStopped(TsbError):
    """a resumable search stopped (time limit or request_stop()) and wrote its checkpoint; `stats` holds the counts so
    far.  Calling the same search again with the same checkpoint continues it."""

    def __init__(self, where: str, stats):
        super().__init__(ESTOPPED, where)
        self.stats = stats


class PfspTables(C.Structure):
    """tsb_pfsp_tables"""
    _fields_ = [
        ("jobs", C.c_int32), ("machines", C.c_int32), ("pairs", C.c_int32),
        ("p_times", C.c_int32 * (MAX_MACHINES * MAX_JOBS)),
        ("min_heads", C.c_int32 * MAX_MACHINES), ("min_tails", C.c_int32 * MAX_MACHINES),
        ("johnson", C.c_int32 * (MAX_PAIRS * MAX_JOBS)), ("lags", C.c_int32 * (MAX_PAIRS * MAX_JOBS)),
        ("mp0", C.c_int32 * MAX_PAIRS), ("mp1", C.c_int32 * MAX_PAIRS), ("mp_order", C.c_int32 * MAX_PAIRS),
    ]


class PfspTables50(C.Structure):
    """tsb_pfsp_tables50 (MAX_JOBS = 50 build)"""
    _fields_ = [
        ("jobs", C.c_int32), ("machines", C.c_int32), ("pairs", C.c_int32),
        ("p_times", C.c_int32 * (MAX_MACHINES * 50)),
        ("min_heads", C.c_int32 * MAX_MACHINES), ("min_tails", C.c_int32 * MAX_MACHINES),
        ("johnson", C.c_int32 * (MAX_PAIRS * 50)), ("lags", C.c_int32 * (MAX_PAIRS * 50)),
        ("mp0", C.c_int32 * MAX_PAIRS), ("mp1", C.c_int32 * MAX_PAIRS), ("mp_order", C.c_int32 * MAX_PAIRS),
    ]


class SearchStats(C.Structure):
    """tsb_search_stats"""
    _fields_ = [
        ("explored_tree", C.c_uint64), ("explored_sol", C.c_uint64), ("best", C.c_int64),
        ("t_step1", C.c_double), ("t_step2", C.c_double), ("t_step3", C.c_double),
        ("offloads", C.c_uint64), ("offloaded_parents", C.c_uint64), ("kernel_launches", C.c_uint64),
        ("per_gpu_tree", C.c_uint64 * 8), ("steals", C.c_uint64),
    ]


# every symbol include/tsb200.h declares: name -> (restype, argtypes)
_vp, _i, _i64, _u64 = C.c_void_p, C.c_int, C.c_int64, C.c_uint64
_pi32 = C.c_void_p
SYMBOLS = {
    "tsb_strerror": (C.c_char_p, [_i]),
    "tsb_last_cuda_error": (C.c_char_p, []),
    "tsb_device_count": (_i, []),
    "tsb_device_sm_count": (_i, [_i]),
    "tsb_init_devices": (_i, [_i]),
    "tsb_bind_thread_to_device": (_i, [_i]),
    "tsb_version": (C.c_char_p, []),
    "tsb_nq_create": (_i, [C.POINTER(_vp), _i, _i, _i, _i]),
    "tsb_nq_create_wide": (_i, [C.POINTER(_vp), _i, _i, _i, _i, _i]),
    "tsb_nq_max_queens": (_i, [_vp]),
    "tsb_nq_destroy": (None, [_vp]),
    "tsb_nq_evaluate": (_i, [_vp, _vp, _i, _vp]),
    "tsb_nq_evaluate_device": (_i, [_vp, _vp, _i, _vp, _vp]),
    "tsb_nq_expand": (_i, [_vp, _vp, _i, _vp, _u64, C.POINTER(_u64), C.POINTER(_u64)]),
    "tsb_nq_expand_device": (_i, [_vp, _vp, _i, _vp, C.POINTER(_u64), C.POINTER(_u64), _vp]),
    "tsb_nq_pool_push": (_i, [_vp, _vp, _i64]),
    "tsb_nq_pool_size": (_i64, [_vp]),
    "tsb_nq_pool_step": (_i, [_vp, _i, _i, C.POINTER(_i64), C.POINTER(_u64), C.POINTER(_u64)]),
    "tsb_nq_pool_drain": (_i, [_vp, _vp, _i64, C.POINTER(_i64)]),
    "tsb_nq_pool_steal": (_i, [_vp, _vp, _i, C.POINTER(_i64)]),
    "tsb_pfsp_pool_steal": (_i, [_vp, _vp, _i, C.POINTER(_i64)]),
    "tsb_nq_pool_run": (_i, [_vp, _i, _i, _i64, C.POINTER(_u64), C.POINTER(_u64), C.POINTER(_u64), C.POINTER(_u64)]),
    "tsb_nq_pool_run_multi": (_i, [C.POINTER(_vp), _i, _i, _i, _i64, C.POINTER(_u64)]),
    "tsb_release_cached_handles": (None, []),
    "tsb_nq_sibling": (_i, [_vp, _i, C.POINTER(_vp)]),
    "tsb_nq_pools_per_launch": (_i, [_vp, _i]),
    "tsb_nq_register_host": (_i, [_vp, _vp, C.c_size_t]),
    "tsb_nq_unregister_host": (_i, [_vp, _vp]),
    "tsb_debug_flag_exchange": (_i, [_i, _i, _i, _i, C.POINTER(C.c_double)]),
    "tsb_nq_set_xfer": (_i, [_vp, _i]),
    "tsb_nq_last_xfer": (_i, [_vp]),
    "tsb_nq_kernel_launches": (_u64, [_vp]),
    "tsb_pfsp_create": (_i, [C.POINTER(_vp), _i, _i, _i, _i, _pi32, _pi32, _pi32, _i, _pi32, _pi32, _pi32, _pi32, _pi32]),
    "tsb_pfsp_create_wide": (_i, [C.POINTER(_vp), _i, _i, _i, _i, _i, _pi32, _pi32, _pi32, _i, _pi32, _pi32, _pi32, _pi32, _pi32]),
    "tsb_pfsp_tables50_build": (_i, [C.POINTER(PfspTables50), _i, _i]),
    "tsb_pfsp_create50_from_tables": (_i, [C.POINTER(_vp), _i, _i, C.POINTER(PfspTables50)]),
    "tsb_pfsp_destroy": (None, [_vp]),
    "tsb_pfsp_evaluate": (_i, [_vp, _i, _vp, _i, _i64, _vp]),
    "tsb_pfsp_evaluate_device": (_i, [_vp, _i, _vp, _i, _i64, _vp, _vp]),
    "tsb_pfsp_expand": (_i, [_vp, _i, _vp, _i, C.POINTER(_i64), _vp, _u64, C.POINTER(_u64), C.POINTER(_u64)]),
    "tsb_pfsp_expand_device": (_i, [_vp, _i, _vp, _i, C.POINTER(_i64), _vp, C.POINTER(_u64), C.POINTER(_u64), _vp]),
    "tsb_pfsp_pool_push": (_i, [_vp, _vp, _i64]),
    "tsb_pfsp_pool_size": (_i64, [_vp]),
    "tsb_pfsp_pool_step": (_i, [_vp, _i, _i, _i, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_u64), C.POINTER(_u64)]),
    "tsb_pfsp_pool_run": (_i, [_vp, _i, _i, _i, _i64, C.POINTER(_i64), C.POINTER(_u64), C.POINTER(_u64), C.POINTER(_u64),
                               C.POINTER(_u64)]),
    "tsb_pfsp_pool_run_multi": (_i, [C.POINTER(_vp), _i, _i, _i, _i, _i64, C.POINTER(_i64), C.POINTER(_u64)]),
    "tsb_pfsp_sibling": (_i, [_vp, _i, C.POINTER(_vp)]),
    "tsb_pfsp_pools_per_launch": (_i, [_vp, _i, _i]),
    "tsb_pfsp_pool_drain": (_i, [_vp, _vp, _i64, C.POINTER(_i64)]),
    "tsb_pfsp_slow_rounds": (_u64, [_vp]),
    "tsb_pfsp_route": (_i, [_vp]),
    "tsb_pfsp_register_host": (_i, [_vp, _vp, C.c_size_t]),
    "tsb_pfsp_unregister_host": (_i, [_vp, _vp]),
    "tsb_pfsp_set_xfer": (_i, [_vp, _i]),
    "tsb_pfsp_last_xfer": (_i, [_vp]),
    "tsb_pfsp_kernel_launches": (_u64, [_vp]),
    "tsb_taillard_nb_jobs": (_i, [_i]),
    "tsb_taillard_nb_machines": (_i, [_i]),
    "tsb_taillard_best_ub": (_i64, [_i]),
    "tsb_pfsp_tables_build": (_i, [C.POINTER(PfspTables), _i]),
    "tsb_pfsp_tables_build_variant": (_i, [C.POINTER(PfspTables), _i, _i]),
    "tsb_pfsp_create_from_tables": (_i, [C.POINTER(_vp), _i, _i, C.POINTER(PfspTables)]),
    "tsb_nq_warmup": (_i, [_i, _i, _vp, _i64, C.POINTER(_i64), C.POINTER(_u64), C.POINTER(_u64)]),
    "tsb_nq_stream": (_vp, [_vp]),
    "tsb_pfsp_stream": (_vp, [_vp]),
    "tsb_nq_search": (_i, [_i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_nq_search_device": (_i, [_i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_nq_search_wide": (_i, [_i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_nq_search_device_wide": (_i, [_i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_pfsp_search": (_i, [_i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_device": (_i, [_i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_nq_search_on": (_i, [_vp, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_on": (_i, [_vp, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_nq_search_device_part": (_i, [_i, _i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_device_part": (_i, [_i, _i, _i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_device_pools": (_i, [_i, _i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_device_pools_part": (_i, [_i, _i, _i, _i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_on_pools": (_i, [_vp, _i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_nq_search_device_ckpt": (_i, [_i, _i, _i, _i, _i, _i, C.c_char_p, C.c_double, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_device_ckpt": (_i, [_i, _i, _i, _i, _i, _i, _i, C.c_char_p, C.c_double, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_wide": (_i, [_i, _i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_device_wide": (_i, [_i, _i, _i, _i, _i, _i, _i, _i, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_device_ckpt_wide": (_i, [_i, _i, _i, _i, _i, _i, _i, _i, C.c_char_p, C.c_double,
                                              C.POINTER(SearchStats)]),
    "tsb_search_request_stop": (None, []),
    "tsb_nq_search_ckpt": (_i, [_i, _i, _i, _i, _i, _i, C.c_char_p, C.c_double, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_ckpt": (_i, [_i, _i, _i, _i, _i, _i, C.c_char_p, C.c_double, C.POINTER(SearchStats)]),
    "tsb_pfsp_search_ckpt_wide": (_i, [_i, _i, _i, _i, _i, _i, _i, C.c_char_p, C.c_double, C.POINTER(SearchStats)]),
}

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                              f"or `make -C {PKG_DIR}` — tsb200 has no CPU fallback")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(code: int, where: str) -> None:
    if code != OK:
        raise TsbError(code, where)


def check_search(code: int, where: str, stats) -> None:
    """check() for the resumable searches: TSB_ESTOPPED raises SearchStopped with the counts so far"""
    if code == ESTOPPED:
        raise SearchStopped(where, stats)
    check(code, where)


def ckpt_args(checkpoint, time_limit):
    """the path and seconds arguments of tsb_*_search[_device]_ckpt (time_limit None: no limit)"""
    return os.fsencode(os.fspath(checkpoint)), -1.0 if time_limit is None else float(time_limit)


def request_stop() -> None:
    """every resumable search running in this process (or the next one to start) stops at its next call boundary
    and writes its checkpoint (tsb_search_request_stop; safe to call from a signal handler)"""
    lib().tsb_search_request_stop()


class Evaluator:
    """What NQueensEvaluator and PfspEvaluator share: the handle's lifecycle and the entry points that take only the
    handle, called as f"{_abi}_<name>" (tsb_nq_* or tsb_pfsp_*)"""

    _abi = ""
    _h = C.c_void_p()
    _owner = None  # a sibling's handle belongs to the evaluator it came from

    def _fn(self, name: str):
        return getattr(lib(), f"{self._abi}_{name}")

    def _check(self, name: str, *args) -> None:
        check(self._fn(name)(self._h, *args), f"{self._abi}_{name}")

    def close(self):
        if self._h and self._owner is None:
            self._fn("destroy")(self._h)
        self._h = C.c_void_p()

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def set_xfer(self, mode: int):
        self._check("set_xfer", mode)

    def register_host(self, arr: np.ndarray) -> None:
        """page-lock + map a long-lived host array (the driver's chunk arrays, allocated once per search) so that
        evaluate_gpu works on it in place; the array must outlive the evaluator or be unregistered"""
        self._check("register_host", arr.ctypes.data, arr.nbytes)

    def unregister_host(self, arr: np.ndarray) -> None:
        self._check("unregister_host", arr.ctypes.data)

    @property
    def kernel_launches(self) -> int:
        return int(self._fn("kernel_launches")(self._h))

    @property
    def last_xfer(self) -> int:
        """route of the last evaluate call: XFER_ROUTE_ZEROCOPY | _PIPELINED | _IN_STAGED | _OUT_STAGED bits"""
        r = int(self._fn("last_xfer")(self._h))
        check(min(r, 0), f"{self._abi}_last_xfer")
        return r

    @property
    def stream(self) -> int:
        """the handle's cudaStream_t (pool / expand / host-buffer entry points launch on it)"""
        return int(self._fn("stream")(self._h) or 0)

    @property
    def pool_size(self) -> int:
        return int(self._fn("pool_size")(self._h))

    @property
    def pool_dtype(self) -> np.dtype:
        """the records of the device pool"""
        return self.node_dtype

    def pool_steal_from(self, victim: "Evaluator", m: int) -> int:
        got = C.c_int64(0)
        check(self._fn("pool_steal")(victim._h, self._h, m, C.byref(got)), f"{self._abi}_pool_steal")
        return int(got.value)

    def pool_drain(self) -> np.ndarray:
        n = self.pool_size
        out = np.empty(max(n, 1), dtype=self.pool_dtype)
        got = C.c_int64(0)
        self._check("pool_drain", out.ctypes.data, n, C.byref(got))
        return out[: got.value].copy()

"""ctypes binding of oracle/liboracle50.so: the CPU oracle (tsb_oracle.c) built with OR_MAX_JOBS = 50, i.e. the
Chapel program as `chpl -sMAX_JOBS=50` would build it (lib/pfsp/PFSP_node.chpl:7): 208-byte nodes, ta031..ta060.
TEST INFRASTRUCTURE ONLY, like everything under oracle/."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import pyoracle as po

MAX_JOBS = 50
MAX_MACHINES = 20
PFSP_NODE_DTYPE = np.dtype([("depth", np.int32), ("limit1", np.int32), ("prmu", np.int32, (MAX_JOBS,))])
assert PFSP_NODE_DTYPE.itemsize == 208


class Tables(C.Structure):
    """or_pfsp_tables with OR_MAX_JOBS = 50"""
    _fields_ = [
        ("jobs", C.c_int32), ("machines", C.c_int32), ("pairs", C.c_int32),
        ("p_times", C.c_int32 * (MAX_MACHINES * MAX_JOBS)),
        ("min_heads", C.c_int32 * MAX_MACHINES), ("min_tails", C.c_int32 * MAX_MACHINES),
        ("johnson", C.c_int32 * (190 * MAX_JOBS)), ("lags", C.c_int32 * (190 * MAX_JOBS)),
        ("mp0", C.c_int32 * 190), ("mp1", C.c_int32 * 190), ("mp_order", C.c_int32 * 190),
    ]

    def arr(self, name, n=None):
        a = np.ctypeslib.as_array(getattr(self, name))
        return a[:n].copy() if n is not None else a.copy()


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        path = os.path.join(po.HERE, "liboracle50.so")
        if not os.path.exists(path):
            po.build(ref=False)
        L = C.CDLL(path)
        L.or_pfsp_tables_build_variant.argtypes = [C.POINTER(Tables), C.c_int, C.c_int, C.c_int]
        L.or_pfsp_tables_from_ptimes.argtypes = [C.POINTER(Tables), C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
        L.or_pfsp_evaluate.argtypes = [C.POINTER(Tables), C.c_int, C.c_void_p, C.c_int, C.c_int64, C.c_void_p]
        L.or_taillard_best_ub.restype = C.c_int64
        _lib = L
    return _lib


def tables(inst: int, heads_mode: int = 0, variant: int = 0) -> Tables:
    t = Tables()
    rc = lib().or_pfsp_tables_build_variant(C.byref(t), inst, heads_mode, variant)
    if rc != 0:
        raise ValueError(f"or_pfsp_tables_build({inst}) -> {rc}")
    return t


def tables_from_ptimes(p_times, heads_mode: int = 0, variant: int = 0) -> Tables:
    """the tables fill_* build from a processing-time matrix p_times[machines, 50] (any values)"""
    return po.tables_from_ptimes(p_times, heads_mode, variant, L=lib(), cls=Tables)


def pfsp_evaluate(t: Tables, lb_kind: int, parents: np.ndarray, best: int, fill: int = -0x32323233) -> np.ndarray:
    assert parents.dtype == PFSP_NODE_DTYPE and parents.flags.c_contiguous
    bounds = np.full(parents.shape[0] * t.jobs, fill, dtype=np.int32)
    lib().or_pfsp_evaluate(C.byref(t), lb_kind, parents.ctypes.data_as(C.c_void_p), parents.shape[0], int(best),
                           bounds.ctypes.data_as(C.c_void_p))
    return bounds


def pfsp_live_mask(parents: np.ndarray, jobs: int) -> np.ndarray:
    return np.arange(jobs)[None, :] >= (parents["limit1"][:, None].astype(np.int64) + 1)

"""ctypes binding of libtsb200_cbase.so (include/tsb200_cbase.h): the reference's C+CUDA `evaluate_gpu` on top of
libtsb200.so, called with torch CUDA tensors for the tables, the parents and the bounds.

    t = tsb200.taillard_tables(14)          # or any struct with the tsb_pfsp_tables fields
    tables = upload_tables(t, "cuda:0")     # the device tables as the reference's drivers build them
    evaluate_gpu(20, LB1, 20 * n, best, tables, parents_d, bounds_d)
    assert status() == 0

Like the C function it returns nothing: a refused call leaves `bounds` unwritten, writes one line to stderr and
sets the sticky code `status()` returns until `release()`.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from ._lib import LB1, LB1_D, LB2, PKG_DIR  # noqa: F401  (the `lb` codes of evaluate_gpu)

LIB_PATH = os.path.join(PKG_DIR, "libtsb200_cbase.so")
_ip = C.POINTER(C.c_int)


class Lb1BoundData(C.Structure):
    """lb1_bound_data (baselines/pfsp/lib/c_bound_simple.h)"""
    _fields_ = [("p_times", _ip), ("min_heads", _ip), ("min_tails", _ip), ("nb_jobs", C.c_int), ("nb_machines", C.c_int)]


class Lb2BoundData(C.Structure):
    """lb2_bound_data (baselines/pfsp/lib/c_bound_johnson.h)"""
    _fields_ = [("johnson_schedules", _ip), ("lags", _ip), ("machine_pairs_1", _ip), ("machine_pairs_2", _ip),
                ("machine_pair_order", _ip), ("nb_machine_pairs", C.c_int), ("nb_jobs", C.c_int), ("nb_machines", C.c_int)]


_lib = None


def lib() -> C.CDLL:
    """libtsb200_cbase.so, loaded once (it finds libtsb200.so next to itself)"""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise OSError(f"{LIB_PATH} is missing: build it with `make -C {PKG_DIR}`")
        L = C.CDLL(LIB_PATH)
        L.evaluate_gpu.restype = None
        L.evaluate_gpu.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, _ip, Lb1BoundData, Lb2BoundData, C.c_void_p,
                                   C.c_void_p]
        L.tsb_cbase_status.restype = C.c_int
        L.tsb_cbase_status.argtypes = []
        L.tsb_cbase_release.restype = None
        L.tsb_cbase_release.argtypes = []
        _lib = L
    return _lib


class DeviceTables:
    """The reference's two bound-data structs over int32 CUDA tensors that this object keeps alive."""

    def __init__(self, tensors: dict, jobs: int, machines: int, pairs: int):
        self.tensors = tensors
        p = {k: C.cast(C.c_void_p(v.data_ptr()), _ip) for k, v in tensors.items()}
        self.lb1 = Lb1BoundData(p["p_times"], p["min_heads"], p["min_tails"], jobs, machines)
        self.lb2 = Lb2BoundData(p["johnson"], p["lags"], p["mp0"], p["mp1"], p["mp_order"], pairs, jobs, machines)


def upload_tables(t, device) -> DeviceTables:
    """Copy the tables of `t` (a ctypes struct with the fields of tsb_pfsp_tables: jobs, machines, pairs, p_times,
    min_heads, min_tails, johnson, lags, mp0, mp1, mp_order) to `device`, one allocation per table as the
    reference's drivers make them."""
    import torch

    jobs, machines, pairs = int(t.jobs), int(t.machines), int(t.pairs)
    sizes = {"p_times": machines * jobs, "min_heads": machines, "min_tails": machines, "johnson": pairs * jobs,
             "lags": pairs * jobs, "mp0": pairs, "mp1": pairs, "mp_order": pairs}
    tensors = {k: torch.from_numpy(np.ctypeslib.as_array(getattr(t, k))[:n].astype(np.int32)).to(device)
               for k, n in sizes.items()}
    return DeviceTables(tensors, jobs, machines, pairs)


def evaluate_gpu(jobs: int, lb: int, size: int, best: int, tables: DeviceTables, parents, bounds,
                 nb_blocks: int = 0) -> None:
    """evaluate_gpu(jobs, lb, size, nbBlocks, &best, lbound1, lbound2, parents, bounds) on the current device of
    `parents` (a CUDA tensor of 88-byte nodes); `bounds` is an int32 CUDA tensor of at least `size` entries.  The
    kernel is queued on the legacy default stream, as the reference's is."""
    import torch

    b = C.c_int(int(best))
    with torch.cuda.device(parents.device):
        lib().evaluate_gpu(int(jobs), int(lb), int(size), int(nb_blocks), C.pointer(b), tables.lb1, tables.lb2,
                           parents.data_ptr(), bounds.data_ptr())


def status() -> int:
    """0, or the first TSB_E* code a call met since the library was loaded or last released"""
    return lib().tsb_cbase_status()


def release() -> None:
    """destroy every cached handle and clear the status"""
    lib().tsb_cbase_release()

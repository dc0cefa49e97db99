"""Return codes of the C ABI (include/tsb200.h) for invalid arguments, on every entry point reachable without a
device: null handles and outputs, negative counts, out-of-range bound kinds and pool counts, and the order in which
the PFSP constructors check their arguments.  Device -1 stands for "no such device" on every machine, with or
without a GPU, so that the constructors' device step is reached the same way everywhere."""
import ctypes as C

import numpy as np
import pytest

import tsb200
from tsb200 import _lib

EINVAL, ENODEV, EUNSUPPORTED = _lib.EINVAL, _lib.ENODEV, _lib.EUNSUPPORTED
NO_DEVICE = -1


@pytest.fixture(scope="module")
def L():
    return tsb200.lib()


def _u64():
    return C.c_uint64(0)


def _i64():
    return C.c_int64(0)


def test_nq_constructors(L):
    h = C.c_void_p()
    assert L.tsb_nq_create(None, 0, 8, 1, 10) == EINVAL
    for N, g, M in ((0, 1, 10), (21, 1, 10), (8, 0, 10), (8, 1, 0), (8, 1, -1)):
        assert L.tsb_nq_create(C.byref(h), 0, N, g, M) == EINVAL, (N, g, M)
    assert L.tsb_nq_create(C.byref(h), NO_DEVICE, 8, 1, 10) == ENODEV
    assert L.tsb_nq_create_wide(None, 0, 24, 8, 1, 10) == EINVAL
    for mq in (20, 23, 25, 0):
        assert L.tsb_nq_create_wide(C.byref(h), 0, mq, 8, 1, 10) == EINVAL, mq
    for N, g, M in ((0, 1, 10), (25, 1, 10), (8, 0, 10), (8, 1, 0)):
        assert L.tsb_nq_create_wide(C.byref(h), 0, 24, N, g, M) == EINVAL, (N, g, M)
    assert L.tsb_nq_create_wide(C.byref(h), NO_DEVICE, 24, 22, 1, 10) == ENODEV
    assert not h


def test_nq_null_handle(L):
    nc, ns, n = _u64(), _u64(), _i64()
    buf = np.zeros(64, dtype=np.uint8)
    L.tsb_nq_destroy(None)
    assert L.tsb_nq_evaluate(None, buf.ctypes.data, 1, buf.ctypes.data) == EINVAL
    assert L.tsb_nq_evaluate_device(None, buf.ctypes.data, 1, buf.ctypes.data, None) == EINVAL
    assert L.tsb_nq_expand(None, buf.ctypes.data, 1, buf.ctypes.data, 64, C.byref(nc), C.byref(ns)) == EINVAL
    assert L.tsb_nq_expand_device(None, buf.ctypes.data, 1, buf.ctypes.data, C.byref(nc), C.byref(ns), None) == EINVAL
    assert L.tsb_nq_pool_push(None, buf.ctypes.data, 1) == EINVAL
    assert L.tsb_nq_pool_size(None) == -1
    assert L.tsb_nq_pool_step(None, 1, 1, C.byref(n), C.byref(nc), C.byref(ns)) == EINVAL
    assert L.tsb_nq_pool_run(None, 1, 1, 1, C.byref(nc), C.byref(nc), C.byref(nc), C.byref(ns)) == EINVAL
    assert L.tsb_nq_pool_drain(None, buf.ctypes.data, 1, C.byref(n)) == EINVAL
    assert L.tsb_nq_pool_steal(None, None, 1, C.byref(n)) == EINVAL
    sib = C.c_void_p()
    assert L.tsb_nq_sibling(None, 1, C.byref(sib)) == EINVAL
    assert L.tsb_nq_pools_per_launch(None, 1000) == 1
    assert L.tsb_nq_register_host(None, buf.ctypes.data, buf.nbytes) == EINVAL
    assert L.tsb_nq_unregister_host(None, buf.ctypes.data) == EINVAL
    assert L.tsb_nq_set_xfer(None, 0) == EINVAL
    assert L.tsb_nq_last_xfer(None) == EINVAL
    assert L.tsb_nq_kernel_launches(None) == 0
    assert L.tsb_nq_stream(None) is None
    assert L.tsb_nq_max_queens(None) == EINVAL


def test_nq_pool_run_multi_arguments(L):
    out = (C.c_uint64 * 32)()
    hs = (C.c_void_p * 8)()
    assert L.tsb_nq_pool_run_multi(None, 1, 1, 1, 1, out) == EINVAL
    for K in (0, -1, 5, 8):
        assert L.tsb_nq_pool_run_multi(hs, K, 1, 1, 1, out) == EINVAL, K
    for K in (1, 4):
        assert L.tsb_nq_pool_run_multi(hs, K, 1, 1, 1, out) == EINVAL, K  # null handles
    assert L.tsb_nq_pool_run_multi(hs, 1, 0, 1, 1, out) == EINVAL
    assert L.tsb_nq_pool_run_multi(hs, 1, 1, 0, 1, out) == EINVAL
    assert L.tsb_nq_pool_run_multi(hs, 1, 1, 1, -1, out) == EINVAL
    assert L.tsb_nq_pool_run_multi(hs, 1, 1, 1, 1, None) == EINVAL


def _pfsp_arrays(jobs, pairs=3, machines=5):
    """well-formed tables of `jobs` jobs: every array the constructors read, as int32 numpy arrays"""
    rng = np.random.default_rng(jobs)
    p = rng.integers(1, 100, size=(machines, jobs)).astype(np.int32)
    heads = np.zeros(machines, np.int32)
    tails = np.zeros(machines, np.int32)
    johnson = np.tile(np.arange(jobs, dtype=np.int32), (max(pairs, 1), 1))
    lags = np.zeros((max(pairs, 1), jobs), np.int32)
    mp0 = np.zeros(max(pairs, 1), np.int32)
    mp1 = np.ones(max(pairs, 1), np.int32)
    order = np.arange(max(pairs, 1), dtype=np.int32)
    return dict(p=p, heads=heads, tails=tails, johnson=johnson, lags=lags, mp0=mp0, mp1=mp1, order=order)


def _ptr(a):
    return None if a is None else a.ctypes.data


def _create(L, wide, out, device, jobs, machines, M, a, pairs, **override):
    args = dict(a)
    args.update(override)
    tail = (_ptr(args["p"]), _ptr(args["heads"]), _ptr(args["tails"]), pairs, _ptr(args["johnson"]),
            _ptr(args["lags"]), _ptr(args["mp0"]), _ptr(args["mp1"]), _ptr(args["order"]))
    if wide is None:
        return L.tsb_pfsp_create(out, device, jobs, machines, M, *tail)
    return L.tsb_pfsp_create_wide(out, device, wide, jobs, machines, M, *tail)


@pytest.mark.parametrize("max_jobs", [None, 20, 50])
def test_pfsp_constructor_check_order(L, max_jobs):
    jobs = 50 if max_jobs == 50 else 20
    a = _pfsp_arrays(jobs)
    h = C.c_void_p()
    out = C.byref(h)

    def rc(out=out, device=NO_DEVICE, jobs=jobs, machines=5, M=10, pairs=3, **kw):
        return _create(L, max_jobs, out, device, jobs, machines, M, a, pairs, **kw)

    # 1. EINVAL: null pointers, M_max < 1, nb_pairs < 0, missing lb2 arrays (ahead of any shape check)
    assert rc(out=None) == EINVAL
    for name in ("p", "heads", "tails"):
        assert rc(**{name: None}) == EINVAL, name
        assert rc(jobs=7, **{name: None}) == EINVAL, name
    for name in ("johnson", "lags", "mp0", "mp1", "order"):
        assert rc(**{name: None}) == EINVAL, name
        assert rc(machines=0, **{name: None}) == EINVAL, name
        assert rc(pairs=0, **{name: None}) == ENODEV, name  # not read without pairs
    for M in (0, -5):
        assert rc(M=M) == EINVAL and rc(M=M, jobs=7) == EINVAL
    assert rc(pairs=-1) == EINVAL and rc(pairs=-1, machines=21) == EINVAL
    # 2. EUNSUPPORTED: job, machine and pair shapes
    for bad in (dict(jobs=jobs - 1), dict(jobs=jobs + 1), dict(machines=0), dict(machines=21), dict(pairs=191)):
        assert rc(**bad) == EUNSUPPORTED, bad
    # 3. the device (ahead of the table indices)
    assert rc() == ENODEV
    assert rc(pairs=0) == ENODEV
    bad_order = a["order"].copy()
    bad_order[1] = 7
    assert rc(order=bad_order) == ENODEV
    bad_john = a["johnson"].copy()
    bad_john[0, 0] = jobs
    assert rc(johnson=bad_john) == ENODEV
    assert not h


def test_pfsp_create_wide_shapes(L):
    a = _pfsp_arrays(50)
    h = C.c_void_p()
    for mj in (0, 21, 49, 51, 100):
        assert _create(L, mj, C.byref(h), NO_DEVICE, 50, 5, 10, a, 3) == EUNSUPPORTED, mj
        assert _create(L, mj, C.byref(h), NO_DEVICE, 50, 5, 0, a, 3) == EINVAL, mj
    assert _create(L, 50, C.byref(h), NO_DEVICE, 20, 5, 10, a, 3) == EUNSUPPORTED


def test_pfsp_null_handle(L):
    nc, ns, n, b = _u64(), _u64(), _i64(), _i64()
    buf = np.zeros(256, dtype=np.uint8)
    d = buf.ctypes.data
    L.tsb_pfsp_destroy(None)
    for lb in (0, 1, 2, 3, -1):
        assert L.tsb_pfsp_evaluate(None, lb, d, 1, 0, d) == EINVAL
        assert L.tsb_pfsp_evaluate_device(None, lb, d, 1, 0, d, None) == EINVAL
        assert L.tsb_pfsp_expand(None, lb, d, 1, C.byref(b), d, 64, C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_pfsp_expand_device(None, lb, d, 1, C.byref(b), d, C.byref(nc), C.byref(ns), None) == EINVAL
        assert L.tsb_pfsp_pool_step(None, lb, 1, 1, C.byref(b), C.byref(n), C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_pfsp_pool_run(None, lb, 1, 1, 1, C.byref(b), C.byref(nc), C.byref(nc), C.byref(nc),
                                   C.byref(ns)) == EINVAL
        assert L.tsb_pfsp_pools_per_launch(None, lb, 1000) == 1
    assert L.tsb_pfsp_pool_push(None, d, 1) == EINVAL
    assert L.tsb_pfsp_pool_size(None) == -1
    assert L.tsb_pfsp_pool_drain(None, d, 1, C.byref(n)) == EINVAL
    assert L.tsb_pfsp_pool_steal(None, None, 1, C.byref(n)) == EINVAL
    sib = C.c_void_p()
    assert L.tsb_pfsp_sibling(None, 1, C.byref(sib)) == EINVAL
    assert L.tsb_pfsp_register_host(None, d, buf.nbytes) == EINVAL
    assert L.tsb_pfsp_unregister_host(None, d) == EINVAL
    assert L.tsb_pfsp_set_xfer(None, 0) == EINVAL
    assert L.tsb_pfsp_last_xfer(None) == EINVAL
    assert L.tsb_pfsp_kernel_launches(None) == 0
    assert L.tsb_pfsp_stream(None) is None
    assert L.tsb_pfsp_slow_rounds(None) == 0
    assert L.tsb_pfsp_route(None) == EINVAL
    t, t50 = _lib.PfspTables(), _lib.PfspTables50()
    h = C.c_void_p()
    assert L.tsb_pfsp_create_from_tables(C.byref(h), 0, 10, None) == EINVAL
    assert L.tsb_pfsp_create50_from_tables(C.byref(h), 0, 10, None) == EINVAL
    assert L.tsb_pfsp_create_from_tables(C.byref(h), 0, 10, C.byref(t)) == EUNSUPPORTED  # jobs = 0
    assert L.tsb_pfsp_create50_from_tables(C.byref(h), 0, 10, C.byref(t50)) == EUNSUPPORTED


def test_pfsp_pool_run_multi_arguments(L):
    out = (C.c_uint64 * 32)()
    best = (C.c_int64 * 8)()
    hs = (C.c_void_p * 8)()
    assert L.tsb_pfsp_pool_run_multi(None, 1, 1, 1, 1, 1, best, out) == EINVAL
    for K in (0, -1, 5, 8):
        assert L.tsb_pfsp_pool_run_multi(hs, K, 1, 1, 1, 1, best, out) == EINVAL, K
    for K in (1, 4):
        assert L.tsb_pfsp_pool_run_multi(hs, K, 1, 1, 1, 1, best, out) == EINVAL, K  # null handles
    for lb in (3, -1):
        assert L.tsb_pfsp_pool_run_multi(hs, 1, lb, 1, 1, 1, best, out) == EINVAL, lb
    assert L.tsb_pfsp_pool_run_multi(hs, 1, 1, 0, 1, 1, best, out) == EINVAL
    assert L.tsb_pfsp_pool_run_multi(hs, 1, 1, 1, 0, 1, best, out) == EINVAL
    assert L.tsb_pfsp_pool_run_multi(hs, 1, 1, 1, 1, -1, best, out) == EINVAL
    assert L.tsb_pfsp_pool_run_multi(hs, 1, 1, 1, 1, 1, None, out) == EINVAL
    assert L.tsb_pfsp_pool_run_multi(hs, 1, 1, 1, 1, 1, best, None) == EINVAL


def test_device_level_entry_points(L):
    cyc = C.c_double(0)
    assert L.tsb_device_sm_count(NO_DEVICE) == 0
    assert L.tsb_debug_flag_exchange(0, 10, 0, 0, None) == EINVAL
    assert L.tsb_debug_flag_exchange(0, 0, 0, 0, C.byref(cyc)) == EINVAL
    assert L.tsb_debug_flag_exchange(NO_DEVICE, 10, 0, 0, C.byref(cyc)) == ENODEV
    assert L.tsb_bind_thread_to_device(NO_DEVICE) == ENODEV

"""Return codes of the C ABI on live handles (`pytest -m gpu`): narrow and 24-queen N-Queens handles, 20-job PFSP
handles (ta014; ta001, whose lb2 takes the one-word-per-use table; one without machine pairs) and 50-job handles
(ta041).  It pins the refusals of the 50-job handle, the table checks and value limits of the PFSP constructors, and
that a sibling pool has its owner's route, bounds and children, whatever the environment says when it is created."""
import ctypes as C

import numpy as np
import pytest

import tsb200
from tsb200 import _lib

pytestmark = pytest.mark.gpu
EINVAL, EUNSUPPORTED, OK = _lib.EINVAL, _lib.EUNSUPPORTED, _lib.OK
INT_MAX = 2**31 - 1
M = 512


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


@pytest.fixture(autouse=True)
def default_routes(monkeypatch):
    monkeypatch.delenv("TSB200_NO_SIMD16", raising=False)
    monkeypatch.delenv("TSB200_NO_LB2U", raising=False)


@pytest.fixture(scope="module")
def L():
    return tsb200.lib()


def tables_without_pairs(inst):
    t = _lib.PfspTables.from_buffer_copy(tsb200.taillard_tables(inst))
    t.pairs = 0
    return t


@pytest.fixture(scope="module")
def pf():
    """the PFSP handles of the module, by name"""
    evs = {"ta014": tsb200.PfspEvaluator(14, M=M), "ta001": tsb200.PfspEvaluator(1, M=M),
           "nopairs": tsb200.PfspEvaluator(tables=tables_without_pairs(14), M=M), "ta041": tsb200.PfspEvaluator(41, M=M)}
    assert evs["ta001"].route & tsb200.ROUTE_LB2U and evs["ta001"].route != evs["ta014"].route
    assert not evs["nopairs"].route & tsb200.ROUTE_LB2 and evs["ta041"].wide
    yield evs
    for ev in evs.values():
        ev.close()


@pytest.fixture(scope="module")
def nq():
    evs = {"narrow": tsb200.NQueensEvaluator(10, M=M), "wide": tsb200.NQueensEvaluator(22, M=M)}
    assert evs["wide"].wide
    yield evs
    for ev in evs.values():
        ev.close()


def rand_nodes(seed, jobs, count):
    rng = np.random.default_rng(seed)
    nodes = np.zeros(count, dtype=tsb200.PFSP_NODE50_DTYPE if jobs > 20 else tsb200.PFSP_NODE_DTYPE)
    depth = rng.integers(0, jobs, size=count)
    nodes["depth"], nodes["limit1"] = depth, depth - 1
    nodes["prmu"][:, :jobs] = np.argsort(rng.random((count, jobs)), axis=1).astype(np.int32)
    return nodes


def u64():
    return C.c_uint64(0)


def i64(v=0):
    return C.c_int64(v)


def test_nq_live_handles(L, nq):
    buf = np.zeros(4096, dtype=np.uint8)
    d = buf.ctypes.data
    for name, ev in nq.items():
        h = ev._h
        nc, ns, n = u64(), u64(), i64()
        assert L.tsb_nq_evaluate(h, d, -1, d) == EINVAL
        assert L.tsb_nq_evaluate(h, d, M + 1, d) == EINVAL
        assert L.tsb_nq_evaluate(h, None, 1, d) == EINVAL and L.tsb_nq_evaluate(h, d, 1, None) == EINVAL
        assert L.tsb_nq_evaluate(h, None, 0, None) == OK
        assert L.tsb_nq_evaluate_device(h, d, -1, d, None) == EINVAL
        assert L.tsb_nq_expand(h, d, -1, d, 64, C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_nq_expand(h, d, 1, d, 64, None, C.byref(ns)) == EINVAL
        assert L.tsb_nq_expand(h, d, 1, d, 64, C.byref(nc), None) == EINVAL
        assert L.tsb_nq_expand_device(h, d, -1, d, C.byref(nc), C.byref(ns), None) == EINVAL
        assert L.tsb_nq_expand_device(h, d, 1, d, None, C.byref(ns), None) == EINVAL
        assert L.tsb_nq_pool_push(h, d, -1) == EINVAL and L.tsb_nq_pool_push(h, None, 1) == EINVAL
        assert L.tsb_nq_pool_step(h, 0, 1, C.byref(n), C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_nq_pool_step(h, 1, M + 1, C.byref(n), C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_nq_pool_step(h, 1, 1, None, C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_nq_pool_run(h, 1, 1, -1, C.byref(nc), C.byref(nc), C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_nq_pool_run(h, 1, 1, 1, None, C.byref(nc), C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_nq_pool_drain(h, d, -1, C.byref(n)) == EINVAL and L.tsb_nq_pool_drain(h, d, 1, None) == EINVAL
        assert L.tsb_nq_pool_steal(h, h, 1, C.byref(n)) == EINVAL
        sib = C.c_void_p()
        for index in (0, -1, 4):
            assert L.tsb_nq_sibling(h, index, C.byref(sib)) == EINVAL, index
        assert L.tsb_nq_sibling(h, 1, None) == EINVAL
        assert L.tsb_nq_set_xfer(h, 3) == EINVAL and L.tsb_nq_set_xfer(h, -1) == EINVAL
        assert L.tsb_nq_register_host(h, None, 16) == EINVAL and L.tsb_nq_register_host(h, d, 0) == EINVAL
        for mode in (0, 1, 2):
            assert L.tsb_nq_set_xfer(h, mode) == OK
        assert L.tsb_nq_pools_per_launch(h, 0) == 1 and L.tsb_nq_pools_per_launch(h, M + 1) == 1
        assert L.tsb_nq_max_queens(h) == (24 if name == "wide" else 20)
    assert nq["wide"].pools_per_launch(M) == 1
    n = i64()
    # a steal between boards of different sizes or record widths is refused
    assert L.tsb_nq_pool_steal(nq["narrow"]._h, nq["wide"]._h, 1, C.byref(n)) == EINVAL
    with tsb200.NQueensEvaluator(11, M=M) as other:
        assert L.tsb_nq_pool_steal(nq["narrow"]._h, other._h, 1, C.byref(n)) == EINVAL
        hs = (C.c_void_p * 2)(nq["narrow"]._h, other._h)
        assert L.tsb_nq_pool_run_multi(hs, 2, 1, 100, 1, (C.c_uint64 * 8)()) == EINVAL
    with tsb200.NQueensEvaluator(10, M=M, max_queens=24) as w10:
        hs = (C.c_void_p * 2)(nq["narrow"]._h, w10._h)
        assert L.tsb_nq_pool_run_multi(hs, 2, 1, 100, 1, (C.c_uint64 * 8)()) == EINVAL
    out = (C.c_uint64 * 8)()
    h = nq["narrow"]._h
    assert L.tsb_nq_pool_run_multi((C.c_void_p * 2)(h, h), 2, 1, 100, 1, out) == EINVAL  # the same pool twice
    assert L.tsb_nq_pool_run_multi((C.c_void_p * 1)(h), 1, 1, M + 1, 1, out) == EINVAL
    assert L.tsb_nq_pool_run_multi((C.c_void_p * 2)(h, None), 2, 1, 100, 1, out) == EINVAL


def test_pfsp_live_handle_arguments(L, pf):
    buf = np.zeros(1 << 16, dtype=np.uint8)
    d = buf.ctypes.data
    for name in ("ta014", "ta001", "nopairs"):
        h = pf[name]._h
        nc, ns, n, b = u64(), u64(), i64(), i64(INT_MAX)
        for lb in (3, -1):
            assert L.tsb_pfsp_evaluate(h, lb, d, 1, 0, d) == EINVAL
            assert L.tsb_pfsp_evaluate_device(h, lb, d, 1, 0, d, None) == EINVAL
            assert L.tsb_pfsp_expand(h, lb, d, 1, C.byref(b), d, 64, C.byref(nc), C.byref(ns)) == EINVAL
            assert L.tsb_pfsp_expand_device(h, lb, d, 1, C.byref(b), d, C.byref(nc), C.byref(ns), None) == EINVAL
            assert L.tsb_pfsp_pool_step(h, lb, 1, 1, C.byref(b), C.byref(n), C.byref(nc), C.byref(ns)) == EINVAL
            assert L.tsb_pfsp_pool_run(h, lb, 1, 1, 1, C.byref(b), C.byref(nc), C.byref(nc), C.byref(nc),
                                       C.byref(ns)) == EINVAL
            assert L.tsb_pfsp_pool_run_multi((C.c_void_p * 1)(h), 1, lb, 1, 1, 1, (C.c_int64 * 1)(), (C.c_uint64 * 4)()) == EINVAL
        assert L.tsb_pfsp_evaluate(h, 1, d, -1, 0, d) == EINVAL and L.tsb_pfsp_evaluate(h, 1, d, M + 1, 0, d) == EINVAL
        assert L.tsb_pfsp_evaluate(h, 1, None, 1, 0, d) == EINVAL and L.tsb_pfsp_evaluate(h, 1, d, 1, 0, None) == EINVAL
        assert L.tsb_pfsp_evaluate(h, 1, None, 0, 0, None) == OK
        assert L.tsb_pfsp_evaluate_device(h, 1, d, -1, 0, d, None) == EINVAL
        assert L.tsb_pfsp_expand(h, 1, d, 1, None, d, 64, C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_pfsp_expand(h, 1, d, M + 1, C.byref(b), d, 64, C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_pfsp_expand_device(h, 1, d, 1, C.byref(b), d, None, C.byref(ns), None) == EINVAL
        assert L.tsb_pfsp_expand_device(h, 1, d, M + 1, C.byref(b), d, C.byref(nc), C.byref(ns), None) == EINVAL
        assert L.tsb_pfsp_pool_push(h, d, -1) == EINVAL and L.tsb_pfsp_pool_push(h, None, 1) == EINVAL
        assert L.tsb_pfsp_pool_step(h, 1, 0, 1, C.byref(b), C.byref(n), C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_pfsp_pool_step(h, 1, 1, M + 1, C.byref(b), C.byref(n), C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_pfsp_pool_step(h, 1, 1, 1, None, C.byref(n), C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_pfsp_pool_run(h, 1, 1, 1, -1, C.byref(b), C.byref(nc), C.byref(nc), C.byref(nc), C.byref(ns)) == EINVAL
        assert L.tsb_pfsp_pool_drain(h, d, -1, C.byref(n)) == EINVAL and L.tsb_pfsp_pool_drain(h, d, 1, None) == EINVAL
        assert L.tsb_pfsp_pool_steal(h, h, 1, C.byref(n)) == EINVAL
        sib = C.c_void_p()
        for index in (0, -1, 4):
            assert L.tsb_pfsp_sibling(h, index, C.byref(sib)) == EINVAL, index
        assert L.tsb_pfsp_set_xfer(h, 3) == EINVAL
        assert L.tsb_pfsp_pools_per_launch(h, 1, 0) == 1 and L.tsb_pfsp_pools_per_launch(h, 1, M + 1) == 1
        # lb2 on a handle without pairs: EINVAL on every entry point, before the count is looked at
        want = EINVAL if name == "nopairs" else OK
        assert L.tsb_pfsp_evaluate(h, 2, None, 0, 0, None) == want
        assert L.tsb_pfsp_evaluate_device(h, 2, None, 0, 0, None, None) == want
        assert L.tsb_pfsp_expand(h, 2, None, 0, C.byref(b), None, 0, C.byref(nc), C.byref(ns)) == want
        assert L.tsb_pfsp_expand_device(h, 2, None, 0, C.byref(b), None, C.byref(nc), C.byref(ns), None) == want
        if name == "nopairs":
            assert L.tsb_pfsp_pool_step(h, 2, 1, 1, C.byref(b), C.byref(n), C.byref(nc), C.byref(ns)) == EINVAL
            assert L.tsb_pfsp_pool_run(h, 2, 1, 1, 1, C.byref(b), C.byref(nc), C.byref(nc), C.byref(nc), C.byref(ns)) == EINVAL
            assert L.tsb_pfsp_pool_run_multi((C.c_void_p * 1)(h), 1, 2, 1, 1, 1, (C.c_int64 * 1)(), (C.c_uint64 * 4)()) == EINVAL
    out, best = (C.c_uint64 * 8)(), (C.c_int64 * 2)()
    h = pf["ta014"]._h
    assert L.tsb_pfsp_pool_run_multi((C.c_void_p * 2)(h, h), 2, 1, 1, 100, 1, best, out) == EINVAL
    assert L.tsb_pfsp_pool_run_multi((C.c_void_p * 2)(h, pf["ta001"]._h), 2, 1, 1, 100, 1, best, out) == EINVAL  # routes
    assert L.tsb_pfsp_pool_run_multi((C.c_void_p * 1)(h), 1, 1, 1, M + 1, 1, best, out) == EINVAL


def test_pfsp_wide_refusals(L, pf):
    """a 50-job handle refuses the fused expand, the device pool and siblings with EUNSUPPORTED, ahead of any other
    argument check; pool_size, pool_drain and pool_steal work on its (empty) pool"""
    w = pf["ta041"]._h
    nc, ns, n, b = u64(), u64(), i64(), i64(INT_MAX)
    d = np.zeros(4096, dtype=np.uint8).ctypes.data
    for lb in (0, 1, 2, 3, -1):
        assert L.tsb_pfsp_expand(w, lb, d, 1, C.byref(b), d, 64, C.byref(nc), C.byref(ns)) == EUNSUPPORTED
        assert L.tsb_pfsp_expand(w, lb, None, -1, None, None, 0, None, None) == EUNSUPPORTED
        assert L.tsb_pfsp_expand_device(w, lb, d, 1, C.byref(b), d, C.byref(nc), C.byref(ns), None) == EUNSUPPORTED
        assert L.tsb_pfsp_expand_device(w, lb, None, -1, None, None, None, None, None) == EUNSUPPORTED
        assert L.tsb_pfsp_pool_step(w, lb, 1, 1, C.byref(b), C.byref(n), C.byref(nc), C.byref(ns)) == EUNSUPPORTED
        assert L.tsb_pfsp_pool_step(w, lb, 0, 0, None, None, None, None) == EUNSUPPORTED
        assert L.tsb_pfsp_pool_run(w, lb, 1, 1, 1, C.byref(b), C.byref(nc), C.byref(nc), C.byref(nc), C.byref(ns)) == EUNSUPPORTED
        assert L.tsb_pfsp_pool_run(w, lb, 0, 0, -1, None, None, None, None, None) == EUNSUPPORTED
        assert L.tsb_pfsp_pools_per_launch(w, lb, 100) == 1
    assert L.tsb_pfsp_pool_push(w, d, 1) == EUNSUPPORTED and L.tsb_pfsp_pool_push(w, None, -1) == EUNSUPPORTED
    sib = C.c_void_p()
    assert L.tsb_pfsp_sibling(w, 1, C.byref(sib)) == EUNSUPPORTED and L.tsb_pfsp_sibling(w, 0, None) == EUNSUPPORTED
    # evaluate keeps the usual checks
    assert L.tsb_pfsp_evaluate(w, 3, d, 1, 0, d) == EINVAL and L.tsb_pfsp_evaluate(w, 1, d, -1, 0, d) == EINVAL
    assert L.tsb_pfsp_evaluate(w, 2, None, 0, 0, None) == OK
    # no wide check on the pool size, drain and steal
    assert L.tsb_pfsp_pool_size(w) == 0
    assert L.tsb_pfsp_pool_drain(w, None, 0, C.byref(n)) == OK and n.value == 0
    assert L.tsb_pfsp_pool_drain(w, d, -1, C.byref(n)) == EINVAL
    with tsb200.PfspEvaluator(42, M=M) as w2:
        assert L.tsb_pfsp_pool_steal(w, w2._h, 1, C.byref(n)) == OK and n.value == 0
    assert L.tsb_pfsp_pool_steal(w, pf["ta014"]._h, 1, C.byref(n)) == EINVAL  # jobs differ
    # run_multi: EUNSUPPORTED when any handle is wide, after the null-handle checks, before device / M_max / route
    out, best = (C.c_uint64 * 16)(), (C.c_int64 * 4)()
    h = pf["ta014"]._h
    for group in ([w], [h, w], [w, h], [h, pf["ta001"]._h, w], [w, w]):
        hs = (C.c_void_p * len(group))(*group)
        assert L.tsb_pfsp_pool_run_multi(hs, len(group), 1, 1, 100, 1, best, out) == EUNSUPPORTED, group
        assert L.tsb_pfsp_pool_run_multi(hs, len(group), 1, 1, M + 1, 1, best, out) == EUNSUPPORTED, group
        assert L.tsb_pfsp_pool_run_multi(hs, len(group), 2, 1, 100, 1, best, out) == EUNSUPPORTED, group
    assert L.tsb_pfsp_pool_run_multi((C.c_void_p * 2)(w, None), 2, 1, 1, 100, 1, best, out) == EUNSUPPORTED
    assert L.tsb_pfsp_pool_run_multi((C.c_void_p * 2)(None, w), 2, 1, 1, 100, 1, best, out) == EINVAL
    assert L.tsb_pfsp_pool_run_multi((C.c_void_p * 2)(h, None), 2, 1, 1, 100, 1, best, out) == EINVAL
    assert L.tsb_pfsp_pool_run_multi((C.c_void_p * 1)(w), 1, 3, 1, 100, 1, best, out) == EINVAL


def modified(inst, edit):
    base = tsb200.taillard_tables50(inst) if inst > 30 else tsb200.taillard_tables(inst)
    t = type(base).from_buffer_copy(base)
    edit(t)
    return t


def create_code(t):
    try:
        tsb200.PfspEvaluator(tables=t, M=16).close()
        return OK
    except tsb200.TsbError as e:
        return e.code


@pytest.mark.parametrize("inst", [14, 41])
def test_pfsp_table_indices(inst):
    jobs = 50 if inst > 30 else 20

    def at(field, i, v):
        def edit(t):
            getattr(t, field)[i] = v
        return edit

    for edit in (at("mp_order", 0, -1), at("mp_order", 3, 10**6), at("mp0", 0, -1), at("mp1", 5, 10), at("mp1", 5, 20),
                 at("johnson", 7, -1), at("johnson", jobs + 3, jobs)):
        assert create_code(modified(inst, edit)) == EINVAL
    assert create_code(modified(inst, lambda t: None)) == OK


def lb2_kept(inst, edit):
    with tsb200.PfspEvaluator(tables=modified(inst, edit), M=16) as ev:
        return bool(ev.route & tsb200.ROUTE_LB2)


@pytest.mark.parametrize("inst", [14, 41])
def test_pfsp_lb2_value_limits(inst):
    """values past a field of the packed lb2 words give a handle without lb2, not an error"""
    jobs = 50 if inst > 30 else 20
    lag_max = 4095 if jobs == 50 else 8191

    def p0(v):
        def edit(t):
            t.p_times[t.johnson[0]] = v  # machine 0 (a machine of some pair), the first job of pair 0's order
        return edit

    def lag(v):
        def edit(t):
            t.lags[3] = v
        return edit

    def tail(v):
        def edit(t):
            t.min_tails[t.mp0[0]] = v
        return edit

    for edit, keep, drop in ((p0, 127, 128), (lag, lag_max, lag_max + 1), (tail, 2047, 2048)):
        assert lb2_kept(inst, edit(keep)), (edit.__name__, keep)
        assert not lb2_kept(inst, edit(drop)), (edit.__name__, drop)
        assert not lb2_kept(inst, edit(-1)), (edit.__name__, -1)


def same_work(a, b, jobs, lbs, seed):
    parents = rand_nodes(seed, jobs, 300)
    for lb in lbs:
        for best in (INT_MAX, 1300):
            assert a.evaluate(parents, lb, best).tobytes() == b.evaluate(parents, lb, best).tobytes(), (lb, best)
            ka, sa, ba = a.expand(parents, lb, best)
            kb, sb, bb = b.expand(parents, lb, best)
            assert (sa, ba) == (sb, bb) and ka.tobytes() == kb.tobytes(), (lb, best)


@pytest.mark.parametrize("name", ["ta014", "ta001", "nopairs"])
def test_sibling_is_its_owner(L, pf, name):
    ev = pf[name]
    lbs = ("lb1", "lb1_d") + (("lb2",) if ev.route & tsb200.ROUTE_LB2 else ())
    for index in (1, 3):
        sib = ev.sibling(index)
        assert sib.route == ev.route
        s = C.c_void_p()
        assert L.tsb_pfsp_sibling(ev._h, index, C.byref(s)) == OK and s.value == sib._h.value
        same_work(ev, sib, 20, lbs, index)
    hs = (C.c_void_p * 2)(ev._h, ev.sibling(1)._h)
    assert L.tsb_pfsp_pool_run_multi(hs, 2, 1, 1, 100, 1, (C.c_int64 * 2)(INT_MAX, INT_MAX), (C.c_uint64 * 8)()) == OK


@pytest.mark.parametrize("var,lost", [("TSB200_NO_SIMD16", tsb200.ROUTE_SIMD16 | tsb200.ROUTE_LB2U),
                                      ("TSB200_NO_LB2U", tsb200.ROUTE_LB2U)])
def test_sibling_keeps_the_route_of_its_owner(monkeypatch, var, lost):
    """the switches are read when a handle is created from tables; a sibling made after they change still takes its
    owner's route"""
    with tsb200.PfspEvaluator(1, M=M) as plain:
        default = plain.route
    assert default & lost == lost
    monkeypatch.setenv(var, "1")
    with tsb200.PfspEvaluator(1, M=M) as owner:
        assert owner.route == default & ~lost
        monkeypatch.delenv(var)
        with tsb200.PfspEvaluator(1, M=M) as fresh:
            assert fresh.route == default
            sib = owner.sibling(2)
            assert sib.route == owner.route
            same_work(owner, sib, 20, ("lb1", "lb1_d", "lb2"), 7)

"""Every host-memory route of the C ABI against the oracle (`pytest -m gpu`): tsb_*_evaluate zero-copy on registered
arrays, copies on one stream, two-stream pipelined copies, staging of unregistered arrays and the fall-back of a
forced zero-copy call; the registry of host ranges; pool_push / pool_drain / expand through the bounce buffers and
through registered arrays; evaluate_device / expand_device on a caller's stream.

Every comparison is bit-exact against oracle.pyoracle / pyoracle50 on live slots.  Every call asserts the route it
took (`last_xfer`).  Every output lives in a larger buffer of sentinel bytes that is checked after each call; a
registered range is the whole buffer, or (`exact`) an array that ends mid-page, so that a read or write past an
array stays inside a page the registration pinned."""
import ctypes as C
import mmap

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po
from oracle import pyoracle50 as po50

pytestmark = pytest.mark.gpu
PAGE = mmap.PAGESIZE
GUARD, FILL = 0xA5, 0x5A
INT_MAX = 2**31 - 1
CHAPEL_MAX = 2**63 - 1
AUTO, MEMCPY, ZEROCOPY = tsb200.XFER_AUTO, tsb200.XFER_MEMCPY, tsb200.XFER_ZEROCOPY
R_ZC, R_PIPE = tsb200.XFER_ROUTE_ZEROCOPY, tsb200.XFER_ROUTE_PIPELINED
R_IN, R_OUT = tsb200.XFER_ROUTE_IN_STAGED, tsb200.XFER_ROUTE_OUT_STAGED
PIPE_CHUNK = 1024
M_MAX = 4096  # a multiple of PIPE_CHUNK
PIPE_COUNTS = (1024, 1025, 2048, 2049, 3073, M_MAX)
REGISTRATIONS = ((False, False), (True, False), (False, True), (True, True))  # (parents, outputs)
ALIGNMENTS = ((0, 0), (8, 0), (0, 4))  # byte shift of (parents, outputs) from a 16-byte boundary
MiB = 1 << 20


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


class Guarded:
    """n records of `dtype` inside a buffer of sentinel bytes, `shift` bytes past a 16-byte boundary with at least 64
    sentinel bytes on either side.  `span` is the range to register: the whole buffer, which ends mid-page, or
    (exact) the records alone, placed so that they end mid-page."""

    def __init__(self, dtype, n, shift=0, exact=False):
        self.dtype = np.dtype(dtype)
        self.nb = n * self.dtype.itemsize
        self.raw = np.full(self.nb + 5 * PAGE, GUARD, dtype=np.uint8)
        base = self.raw.ctypes.data
        page0 = -base % PAGE
        if exact:
            lo = page0 + PAGE + (PAGE // 2 - self.nb) % PAGE
            lo -= (base + lo) % 16
            self.off, hi = lo, lo + self.nb
        else:
            lo = page0 + 64
            self.off = lo + 64 + shift
            hi = self.off + self.nb + 64
            hi += (PAGE // 2 - (base + hi)) % PAGE
        assert 16 <= (base + hi) % PAGE <= PAGE - 16
        self.lo, self.hi = lo, hi
        self.span = self.raw[lo:hi]
        self.bytes = self.raw[self.off:self.off + self.nb]
        self.data = self.bytes.view(self.dtype)

    @property
    def ptr(self):
        return self.raw.ctypes.data + self.off

    def guards_ok(self):
        return bool((self.raw[:self.off] == GUARD).all() and (self.raw[self.off + self.nb:] == GUARD).all())


def route_of(mode, reg_in, reg_out, aligned, count, pipe_min=1, pipe_chunk=PIPE_CHUNK):
    """the route a tsb_*_evaluate call is meant to take"""
    if reg_in and reg_out and aligned and mode != MEMCPY:
        return R_ZC
    return ((R_PIPE if count >= pipe_min and count > pipe_chunk else 0) | (0 if reg_in else R_IN)
            | (0 if reg_out else R_OUT))


def rand_nq(rng, N, count):
    nodes = np.zeros(count, dtype=tsb200.NQ_NODE_DTYPE)
    nodes["depth"] = rng.integers(0, N + 1, size=count)
    nodes["board"][:, :N] = np.argsort(rng.random((count, N)), axis=1).astype(np.uint8)
    return nodes


def rand_pfsp(rng, jobs, count, dtype=tsb200.PFSP_NODE_DTYPE):
    nodes = np.zeros(count, dtype=dtype)
    depth = rng.integers(1, jobs, size=count)
    nodes["depth"], nodes["limit1"] = depth, depth - 1
    nodes["prmu"][:, :jobs] = np.argsort(rng.random((count, jobs)), axis=1).astype(np.int32)
    return nodes


def copy_tables(src, cls):
    t = cls()
    for name in ("jobs", "machines", "pairs"):
        setattr(t, name, getattr(src, name))
    for name in ("p_times", "min_heads", "min_tails", "johnson", "lags", "mp0", "mp1", "mp_order"):
        np.ctypeslib.as_array(getattr(t, name))[:] = np.ctypeslib.as_array(getattr(src, name))
    return t


class Problem:
    """one handle's evaluate call and its oracle: parents (M records) -> want, live (M x width)"""

    def __init__(self, ev, parents, width, out_dtype, call, want, live):
        self.ev, self.parents, self.width, self.out_dtype = ev, parents, width, out_dtype
        self.parent_bytes = parents.view(np.uint8)
        self.call = call  # call(parents_ptr, count, out_ptr) -> tsb status
        self.want_live = np.where(live, want, 0)
        self.live = live

    def check(self, out, count, err):
        got = out.data[: count * self.width].reshape(count, self.width)
        assert np.array_equal(np.where(self.live[:count], got, 0), self.want_live[:count]), err
        assert (out.bytes[count * self.width * out.dtype.itemsize:] == FILL).all(), f"{err}: written past count"
        assert out.guards_ok(), f"{err}: sentinels overwritten"


def nq_problem(ev, N, M, seed):
    parents = rand_nq(np.random.default_rng(seed), N, M)
    want = po.nq_evaluate(parents.view(po.NQ_NODE_DTYPE), N).reshape(M, N)
    live = po.nq_live_mask(parents.view(po.NQ_NODE_DTYPE), N)
    call = lambda p, n, o: tsb200.lib().tsb_nq_evaluate(ev._h, p, n, o)  # noqa: E731
    return Problem(ev, parents, N, np.uint8, call, want, live)


def pfsp_problem(ev, lb, best, M, seed):
    rng = np.random.default_rng(seed)
    kind = tsb200.LB_NAMES[lb]
    if ev.wide:
        parents = rand_pfsp(rng, 50, M, tsb200.PFSP_NODE50_DTYPE)
        t = copy_tables(ev.tables, po50.Tables)
        want = po50.pfsp_evaluate(t, kind, parents.view(po50.PFSP_NODE_DTYPE), min(best, 2**62))
        live = po50.pfsp_live_mask(parents.view(po50.PFSP_NODE_DTYPE), 50)
    else:
        parents = rand_pfsp(rng, 20, M)
        t = copy_tables(ev.tables, po.Tables)
        want = po.pfsp_evaluate(t, kind, parents.view(po.PFSP_NODE_DTYPE), best)
        live = po.pfsp_live_mask(parents.view(po.PFSP_NODE_DTYPE), 20)
    call = lambda p, n, o: tsb200.lib().tsb_pfsp_evaluate(ev._h, kind, p, n, int(best), o)  # noqa: E731
    return Problem(ev, parents, ev.jobs, np.int32, call, want.reshape(M, ev.jobs), live)


def run_call(pb, pin, out, count, mode, want_route, tag):
    ev = pb.ev
    out.bytes[:] = FILL
    l0 = ev.kernel_launches
    rc = pb.call(pin.ptr, count, out.ptr)
    err = f"{tag} mode={mode} count={count}"
    assert rc == 0, f"{err}: status {rc}"
    assert ev.last_xfer == want_route, f"{err}: route {ev.last_xfer}, meant {want_route}"
    launches = -(-count // PIPE_CHUNK) if want_route & R_PIPE else 1
    assert ev.kernel_launches - l0 == launches, err
    pb.check(out, count, err)
    assert pin.guards_ok() and np.array_equal(pin.bytes, pb.parent_bytes), f"{err}: parents changed"


def route_matrix(pb, tile):
    """every registration x alignment x transfer mode x count of one handle made with TSB200_PIPE_MIN=1 and
    TSB200_PIPE_CHUNK=1024, and count == M_max on arrays that end mid-page"""
    ev, M = pb.ev, pb.parents.shape[0]
    assert M == M_MAX
    counts = (1, tile - 1, tile, tile + 1) + PIPE_COUNTS
    for reg_in, reg_out in REGISTRATIONS:
        for sh_in, sh_out in ALIGNMENTS:
            pin = Guarded(pb.parents.dtype, M, sh_in)
            out = Guarded(pb.out_dtype, M * pb.width, sh_out)
            pin.data[:] = pb.parents
            regs = [b for b, r in ((pin, reg_in), (out, reg_out)) if r]
            for b in regs:
                ev.register_host(b.span)
            for mode in (AUTO, MEMCPY, ZEROCOPY):
                ev.set_xfer(mode)
                for count in counts:
                    want = route_of(mode, reg_in, reg_out, sh_in == sh_out == 0, count)
                    run_call(pb, pin, out, count, mode, want, f"registered={reg_in, reg_out} shift={sh_in, sh_out}")
            for b in regs:
                ev.unregister_host(b.span)
        # the driver's case: arrays of exactly M_max records, registered as they are
        pin = Guarded(pb.parents.dtype, M, exact=True)
        out = Guarded(pb.out_dtype, M * pb.width, exact=True)
        pin.data[:] = pb.parents
        regs = [b for b, r in ((pin, reg_in), (out, reg_out)) if r]
        for b in regs:
            ev.register_host(b.span)
        for mode in (AUTO, MEMCPY, ZEROCOPY):
            ev.set_xfer(mode)
            run_call(pb, pin, out, M, mode, route_of(mode, reg_in, reg_out, True, M), f"exact registered={reg_in, reg_out}")
        for b in regs:
            ev.unregister_host(b.span)
    ev.set_xfer(AUTO)


@pytest.fixture
def pipelined(monkeypatch):
    monkeypatch.setenv("TSB200_PIPE_MIN", "1")
    monkeypatch.setenv("TSB200_PIPE_CHUNK", str(PIPE_CHUNK))


# ------------------------------------------------------------------------------------------ evaluate routes
@pytest.mark.parametrize("kernel", ["small", "tma"])
@pytest.mark.parametrize("N", [4, 17, 20])
def test_nq_evaluate_routes(N, kernel, pipelined, monkeypatch):
    if kernel == "tma":
        monkeypatch.setenv("TSB200_NQ_TILE_THREADS", "128")  # the TMA-pipelined kernel at every chunk size
    with tsb200.NQueensEvaluator(N, M=M_MAX) as ev:
        route_matrix(nq_problem(ev, N, M_MAX, 100 + N), 128 if kernel == "small" else 512)


@pytest.mark.parametrize("inst", [1, 14, 21])  # 5, 10 and 20 template machines
def test_pfsp_evaluate_routes(inst, pipelined):
    opt = int(tsb200.lib().tsb_taillard_best_ub(inst))
    with tsb200.PfspEvaluator(inst, M=M_MAX) as ev:
        for lb, best, tile in (("lb1", opt, 128), ("lb1_d", opt, 128), ("lb2", INT_MAX, 64), ("lb2", opt, 64)):
            route_matrix(pfsp_problem(ev, lb, best, M_MAX, inst), tile)


@pytest.mark.parametrize("inst", [31, 41, 51])  # 50 jobs; 5, 10 and 20 machines
def test_pfsp50_evaluate_routes(inst, pipelined):
    opt = int(tsb200.lib().tsb_taillard_best_ub(inst))
    with tsb200.PfspEvaluator(inst, M=M_MAX) as ev:
        assert ev.wide
        for lb, best in (("lb1", opt), ("lb1_d", opt), ("lb2", INT_MAX), ("lb2", opt)):
            route_matrix(pfsp_problem(ev, lb, best, M_MAX, inst), 64)
        # count > M_max is refused, not truncated
        big = np.zeros(M_MAX + 1, dtype=tsb200.PFSP_NODE50_DTYPE)
        with pytest.raises(tsb200.TsbError) as e:
            ev.evaluate(big, "lb1", opt)
        assert e.value.code == -1


DEFAULT_COUNT = 262145  # one record past the default pipe_chunk (262 144), above pipe_min (131 072)


@pytest.mark.parametrize("problem", ["nq17", "ta014", "ta041"])
def test_default_thresholds(problem):
    """the default thresholds: staged copies in two sub-chunks, and zero-copy on the same data"""
    n = DEFAULT_COUNT
    if problem == "nq17":
        ev = tsb200.NQueensEvaluator(17, M=n)
        parents = rand_nq(np.random.default_rng(5), 17, n)
        width, out_dtype, call = 17, np.uint8, lambda p, o: ev.evaluate_gpu(p, n * 17, o)
        sample = np.arange(n)
        want = po.nq_evaluate(parents.view(po.NQ_NODE_DTYPE), 17).reshape(-1, 17)
        live = po.nq_live_mask(parents.view(po.NQ_NODE_DTYPE), 17)
    else:
        inst = int(problem[2:])
        ev = tsb200.PfspEvaluator(inst, M=n)
        opt = int(tsb200.lib().tsb_taillard_best_ub(inst))
        parents = rand_pfsp(np.random.default_rng(inst), ev.jobs, n, ev.node_dtype)
        width, out_dtype, call = ev.jobs, np.int32, lambda p, o: ev.evaluate_gpu(p, n * ev.jobs, opt, "lb1", o)
        sample = np.append(np.arange(0, n, 61), n - 1)  # every 61st record and the last one
        sub = np.ascontiguousarray(parents[sample])
        if ev.wide:
            t = copy_tables(ev.tables, po50.Tables)
            want = po50.pfsp_evaluate(t, 1, sub.view(po50.PFSP_NODE_DTYPE), opt).reshape(-1, width)
            live = po50.pfsp_live_mask(sub.view(po50.PFSP_NODE_DTYPE), width)
        else:
            t = copy_tables(ev.tables, po.Tables)
            want = po.pfsp_evaluate(t, 1, sub.view(po.PFSP_NODE_DTYPE), opt).reshape(-1, width)
            live = po.pfsp_live_mask(sub.view(po.PFSP_NODE_DTYPE), width)
    live_full = live_all(parents, width, ev)
    with ev:
        outs = []
        for registered in (False, True):
            pin, out = Guarded(parents.dtype, n), Guarded(out_dtype, n * width)
            pin.data[:] = parents
            out.bytes[:] = FILL
            if registered:
                ev.register_host(pin.span)
                ev.register_host(out.span)
            l0 = ev.kernel_launches
            call(pin.data, out.data)
            if registered:
                assert ev.last_xfer == R_ZC and ev.kernel_launches - l0 == 1
                ev.unregister_host(pin.span)
                ev.unregister_host(out.span)
            else:
                assert ev.last_xfer == R_PIPE | R_IN | R_OUT and ev.kernel_launches - l0 == 2
            assert out.guards_ok() and pin.guards_ok()
            got = out.data.reshape(-1, width)
            np.testing.assert_array_equal(got[sample][live], want[live], err_msg=f"registered={registered}")
            outs.append(np.where(live_full, got, 0))
        np.testing.assert_array_equal(outs[0], outs[1])


def live_all(parents, width, ev):
    if isinstance(ev, tsb200.NQueensEvaluator):
        return po.nq_live_mask(parents.view(po.NQ_NODE_DTYPE), width)
    return np.arange(width)[None, :] >= (parents["limit1"][:, None].astype(np.int64) + 1)


# ------------------------------------------------------------------------------------------ the registry
def nq_eval_into(ev, pin, out, count, N):
    out.bytes[:] = FILL
    tsb200.check(tsb200.lib().tsb_nq_evaluate(ev._h, pin.ptr, count, out.ptr), "tsb_nq_evaluate")
    par = np.ascontiguousarray(pin.data[:count])
    want = po.nq_evaluate(par.view(po.NQ_NODE_DTYPE), N).reshape(-1, N)
    live = po.nq_live_mask(par.view(po.NQ_NODE_DTYPE), N)
    got = out.data[: count * N].reshape(-1, N)
    np.testing.assert_array_equal(got[live], want[live])
    assert (out.bytes[count * N:] == FILL).all() and out.guards_ok()
    return ev.last_xfer


def test_registry_rules():
    N, n = 8, 256
    rng = np.random.default_rng(9)
    with tsb200.NQueensEvaluator(N, M=n) as ev:
        pin, out = Guarded(tsb200.NQ_NODE_DTYPE, n), Guarded(np.uint8, n * N)
        pin.data[:] = rand_nq(rng, N, n)
        ev.register_host(pin.span)
        ev.register_host(pin.span)          # the same range again: nothing to do
        ev.register_host(pin.span[64:600])  # a range inside it: nothing to do
        ev.register_host(out.span)
        assert nq_eval_into(ev, pin, out, n, N) == R_ZC
        # partly overlapping ranges, on either side
        for bad in (pin.raw[pin.lo - 32:pin.lo + 16], pin.raw[pin.lo + 100:pin.hi + 32]):
            with pytest.raises(tsb200.TsbError) as e:
                ev.register_host(bad)
            assert e.value.code == -1
        # unregistering: only the pointer a range was registered with, and only once
        with pytest.raises(tsb200.TsbError) as e:
            ev.unregister_host(pin.span[16:])
        assert e.value.code == -1
        ev.unregister_host(pin.span)
        assert nq_eval_into(ev, pin, out, n, N) == R_IN
        with pytest.raises(tsb200.TsbError) as e:
            ev.unregister_host(pin.span)
        assert e.value.code == -1
        ev.unregister_host(out.span)
        assert nq_eval_into(ev, pin, out, n, N) == R_IN | R_OUT


def test_registry_range_straddles_the_end():
    """a call whose parents start inside a registered range and end past it (inside the same page) is staged"""
    N, n = 8, 64
    rng = np.random.default_rng(10)
    with tsb200.NQueensEvaluator(N, M=n) as ev:
        pin, out = Guarded(tsb200.NQ_NODE_DTYPE, n), Guarded(np.uint8, n * N)
        pin.data[:] = rand_nq(rng, N, n)
        base = pin.raw.ctypes.data
        head = pin.raw[pin.lo:pin.off + 21 * (n // 2) + 5]  # ends inside a record in the middle of the parents
        assert (base + pin.off + 21 * (n // 2) + 4) // PAGE == (base + pin.off + 21 * n - 1) // PAGE  # same page
        ev.register_host(head)
        ev.register_host(out.span)
        for mode in (AUTO, ZEROCOPY, MEMCPY):
            ev.set_xfer(mode)
            assert nq_eval_into(ev, pin, out, n, N) == R_IN, mode
            assert nq_eval_into(ev, pin, out, n // 4, N) == (R_ZC if mode != MEMCPY else 0), mode
        ev.unregister_host(head)
        ev.unregister_host(out.span)


def test_registry_disabled(monkeypatch):
    monkeypatch.setenv("TSB200_NO_REGISTER", "1")  # register_host does nothing: every call is staged
    N, n = 12, 1000
    with tsb200.NQueensEvaluator(N, M=n) as ev:
        pin, out = Guarded(tsb200.NQ_NODE_DTYPE, n), Guarded(np.uint8, n * N)
        pin.data[:] = rand_nq(np.random.default_rng(11), N, n)
        ev.register_host(pin.span)
        ev.register_host(out.span)
        for mode in (AUTO, ZEROCOPY, MEMCPY):
            ev.set_xfer(mode)
            assert nq_eval_into(ev, pin, out, n, N) == R_IN | R_OUT
        ev.unregister_host(pin.span)
        ev.unregister_host(out.span)


@pytest.mark.parametrize("problem", ["nq", "pfsp"])
def test_registry_two_arrays_in_one_page(problem):
    """a driver's two small chunk arrays that share a page: both are registered and evaluated in place, in any order
    of unregistering"""
    n = 16
    raw = np.full(4 * PAGE, GUARD, dtype=np.uint8)
    page = raw[-raw.ctypes.data % PAGE:][PAGE:2 * PAGE]  # one whole page of the buffer
    rng = np.random.default_rng(12)
    if problem == "nq":
        N = 8
        ev = tsb200.NQueensEvaluator(N, M=n)
        parents = page[64:64 + 21 * n].view(tsb200.NQ_NODE_DTYPE)
        parents[:] = rand_nq(rng, N, n)
        out = page[1024:1024 + N * n]
        width, out_dtype = N, np.uint8
        want = po.nq_evaluate(np.ascontiguousarray(parents).view(po.NQ_NODE_DTYPE), N).reshape(n, N)
        live = po.nq_live_mask(np.ascontiguousarray(parents).view(po.NQ_NODE_DTYPE), N)
        run = lambda: ev.evaluate_gpu(parents, n * N, out)  # noqa: E731
    else:
        ev = tsb200.PfspEvaluator(14, M=n)
        parents = page[64:64 + 88 * n].view(tsb200.PFSP_NODE_DTYPE)
        parents[:] = rand_pfsp(rng, 20, n)
        out = page[2048:2048 + 80 * n].view(np.int32)
        width, out_dtype = 20, np.int32
        want = po.pfsp_evaluate(copy_tables(ev.tables, po.Tables), 1, np.ascontiguousarray(parents).view(po.PFSP_NODE_DTYPE),
                                1377).reshape(n, 20)
        live = po.pfsp_live_mask(np.ascontiguousarray(parents).view(po.PFSP_NODE_DTYPE), 20)
        run = lambda: ev.evaluate_gpu(parents, n * 20, 1377, "lb1", out)  # noqa: E731

    def check(route):
        out.view(np.uint8)[:] = FILL
        run()
        assert ev.last_xfer == route
        np.testing.assert_array_equal(out.reshape(n, width)[live], want[live])

    with ev:
        ev.register_host(parents)
        ev.register_host(out)
        check(R_ZC)
        ev.unregister_host(parents)  # the page stays locked for `out`
        check(R_IN)
        ev.register_host(parents)
        check(R_ZC)
        ev.unregister_host(out)
        check(R_OUT)
        ev.unregister_host(parents)
        check(R_IN | R_OUT)
    assert (raw[:page.ctypes.data - raw.ctypes.data + 64] == GUARD).all()


# ------------------------------------------------------------------------------------------ bounced / registered copies
def piece_edge_sizes(rec):
    """pools of 1 MiB - 1 record .. 1 MiB + 1 record (the first bounce-piece boundary), of 2 MiB (two pieces, and one
    record more: a third piece, the first to wait for its buffer's event) and above 3 MiB"""
    m = MiB // rec
    return sorted({m - 1, m, m + 1, 2 * MiB // rec, 2 * MiB // rec + 1, 7 * MiB // 2 // rec})


@pytest.mark.parametrize("problem", ["nq", "pfsp"])
def test_pool_push_drain_piece_edges(problem):
    rng = np.random.default_rng(13)
    if problem == "nq":
        N = 17
        ev = tsb200.NQueensEvaluator(N, M=1000)
        make, dtype = (lambda n: rand_nq(rng, N, n)), tsb200.NQ_NODE_DTYPE
        drain = tsb200.lib().tsb_nq_pool_drain
    else:
        ev = tsb200.PfspEvaluator(14, M=1000)
        make, dtype = (lambda n: rand_pfsp(rng, 20, n)), tsb200.PFSP_NODE_DTYPE
        drain = tsb200.lib().tsb_pfsp_pool_drain
    with ev:
        for n in piece_edge_sizes(dtype.itemsize):
            nodes = make(n)
            for registered in (False, True):
                src, dst = Guarded(dtype, n, shift=8), Guarded(dtype, n, shift=4)
                src.data[:] = nodes
                dst.bytes[:] = FILL
                if registered:
                    ev.register_host(src.span)
                    ev.register_host(dst.span)
                ev.pool_push(src.data)
                assert ev.pool_size == n
                got = C.c_int64(0)
                tsb200.check(drain(ev._h, dst.ptr, n, C.byref(got)), "pool_drain")
                assert got.value == n and ev.pool_size == 0
                assert dst.bytes.tobytes() == nodes.tobytes(), f"n={n} registered={registered}"
                assert dst.guards_ok() and src.guards_ok()
                if registered:
                    ev.unregister_host(src.span)
                    ev.unregister_host(dst.span)


def expand_call(ev, pb_kind, pin, count, out, cap, best):
    nc, ns = C.c_uint64(0), C.c_uint64(0)
    if pb_kind == "nq":
        rc = tsb200.lib().tsb_nq_expand(ev._h, pin.ptr, count, out.ptr, cap, C.byref(nc), C.byref(ns))
        return rc, nc.value, ns.value, None
    b = C.c_int64(best)
    rc = tsb200.lib().tsb_pfsp_expand(ev._h, 1, pin.ptr, count, C.byref(b), out.ptr, cap, C.byref(nc), C.byref(ns))
    return rc, nc.value, ns.value, b.value


@pytest.mark.parametrize("problem", ["nq", "pfsp"])
def test_host_expand_children_arrays(problem):
    """host expand into registered and unregistered children arrays (several bounce pieces), and a children array
    one node too small: TSB_ENOMEM with the counts set and the array untouched"""
    rng = np.random.default_rng(14)
    count = 20000
    if problem == "nq":
        N = 17
        ev = tsb200.NQueensEvaluator(N, M=count)
        parents = rand_nq(rng, N, count)
        parents["depth"] = rng.integers(0, 7, size=count)
        kids, sol = po.nq_expand(parents.view(po.NQ_NODE_DTYPE), N)
        best_after, dtype, best = None, tsb200.NQ_NODE_DTYPE, None
    else:
        count = 5000
        ev = tsb200.PfspEvaluator(14, M=count)
        parents = rand_pfsp(rng, 20, count)
        parents["depth"] = np.minimum(parents["depth"], 18)  # no leaves: best stays, every child is kept
        parents["limit1"] = parents["depth"] - 1
        best = INT_MAX
        kids, sol, best_after = po.pfsp_expand(copy_tables(ev.tables, po.Tables), 1, parents.view(po.PFSP_NODE_DTYPE), best)
        dtype = tsb200.PFSP_NODE_DTYPE
    n = kids.shape[0]
    assert n * dtype.itemsize > 2 * MiB
    with ev:
        for registered in (False, True):
            pin, out = Guarded(dtype, count, shift=8), Guarded(dtype, n + 8, shift=4)
            pin.data[:] = parents
            if registered:
                ev.register_host(pin.span)
                ev.register_host(out.span)
            for cap, status in ((n - 1, -3), (n, 0)):
                out.bytes[:] = FILL
                rc, nc, ns, b = expand_call(ev, problem, pin, count, out, cap, best)
                assert (rc, nc, ns) == (status, n, sol), (registered, cap)
                if problem == "pfsp":
                    assert b == best_after
                if status:
                    assert (out.bytes == FILL).all(), "a refused expand wrote children"
                else:
                    assert out.bytes[: n * dtype.itemsize].tobytes() == kids.tobytes()
                    assert (out.bytes[n * dtype.itemsize:] == FILL).all()
                assert out.guards_ok() and pin.guards_ok()
            if registered:
                ev.unregister_host(pin.span)
                ev.unregister_host(out.span)


# ------------------------------------------------------------------------------------------ caller streams
SLEEP = 20_000_000  # cycles (~10 ms) the side stream spends before the parents are written


def device_parents(torch, nodes, stale):
    """(the stream-ordered source of the parents: x, key with x ^ key = nodes; a device buffer holding `stale`)"""
    dev = torch.device("cuda:0")
    b = torch.from_numpy(nodes.view(np.uint8).copy()).to(dev)
    key = torch.randint(0, 256, b.shape, dtype=torch.uint8, device=dev)
    d_par = torch.from_numpy(stale.view(np.uint8).copy()).to(dev)
    torch.cuda.synchronize()
    return b ^ key, key, d_par


def test_nq_evaluate_device_on_caller_stream():
    import torch
    N, n = 17, 3000
    rng = np.random.default_rng(15)
    nodes, stale = rand_nq(rng, N, n), rand_nq(rng, N, n)
    want = po.nq_evaluate(nodes.view(po.NQ_NODE_DTYPE), N).reshape(n, N)
    live = po.nq_live_mask(nodes.view(po.NQ_NODE_DTYPE), N)
    with tsb200.NQueensEvaluator(N, M=n) as ev:
        for which in ("side", "handle"):
            s = torch.cuda.Stream() if which == "side" else torch.cuda.ExternalStream(ev.stream)
            x, key, d_par = device_parents(torch, nodes, stale)
            d_out = torch.full((n * N,), FILL, dtype=torch.uint8, device="cuda:0")
            torch.cuda.synchronize()
            with torch.cuda.stream(s):
                torch.cuda._sleep(SLEEP)
                torch.bitwise_xor(x, key, out=d_par)
                ev.evaluate_device(d_par.data_ptr(), n, d_out.data_ptr(), s.cuda_stream if which == "side" else 0)
                got = d_out.cpu().numpy().reshape(n, N)  # ordered on s; waits for s alone
            np.testing.assert_array_equal(got[live], want[live], err_msg=which)


@pytest.mark.parametrize("inst", [14, 41])
def test_pfsp_evaluate_device_on_caller_stream(inst):
    import torch
    n = 3000
    rng = np.random.default_rng(16)
    opt = int(tsb200.lib().tsb_taillard_best_ub(inst))
    with tsb200.PfspEvaluator(inst, M=n) as ev:
        jobs = ev.jobs
        nodes, stale = rand_pfsp(rng, jobs, n, ev.node_dtype), rand_pfsp(rng, jobs, n, ev.node_dtype)
        if ev.wide:
            want = po50.pfsp_evaluate(copy_tables(ev.tables, po50.Tables), 2, nodes.view(po50.PFSP_NODE_DTYPE), opt)
        else:
            want = po.pfsp_evaluate(copy_tables(ev.tables, po.Tables), 2, nodes.view(po.PFSP_NODE_DTYPE), opt)
        want = want.reshape(n, jobs)
        live = live_all(nodes, jobs, ev)
        for which in ("side", "handle"):
            s = torch.cuda.Stream() if which == "side" else torch.cuda.ExternalStream(tsb200.lib().tsb_pfsp_stream(ev._h))
            x, key, d_par = device_parents(torch, nodes, stale)
            d_out = torch.full((n * jobs,), -1, dtype=torch.int32, device="cuda:0")
            torch.cuda.synchronize()
            with torch.cuda.stream(s):
                torch.cuda._sleep(SLEEP)
                torch.bitwise_xor(x, key, out=d_par)
                ev.evaluate_device("lb2", d_par.data_ptr(), n, opt, d_out.data_ptr(), s.cuda_stream if which == "side" else 0)
                got = d_out.cpu().numpy().reshape(n, jobs)
            np.testing.assert_array_equal(got[live], want[live], err_msg=which)


def test_nq_expand_device_every_child_offset():
    """children at every byte offset 0..15, written on the caller's stream after the parents are, guards after them"""
    import torch
    N, n = 14, 2000
    rng = np.random.default_rng(17)
    nodes, stale = rand_nq(rng, N, n), rand_nq(rng, N, n)
    kids, sol = po.nq_expand(nodes.view(po.NQ_NODE_DTYPE), N)
    kb = kids.tobytes()
    with tsb200.NQueensEvaluator(N, M=n) as ev:
        for off in range(16):
            s = torch.cuda.Stream()
            x, key, d_par = device_parents(torch, nodes, stale)
            d_kids = torch.full((len(kb) + 16 + 64,), GUARD, dtype=torch.uint8, device="cuda:0")
            torch.cuda.synchronize()
            with torch.cuda.stream(s):
                torch.cuda._sleep(SLEEP // 4)
                torch.bitwise_xor(x, key, out=d_par)
                nc, ns = ev.expand_device(d_par.data_ptr(), n, d_kids.data_ptr() + off, s.cuda_stream)
                got = d_kids.cpu().numpy()
            assert (nc, ns) == (kids.shape[0], sol), off
            assert got[off:off + len(kb)].tobytes() == kb, off
            assert (got[:off] == GUARD).all() and (got[off + len(kb):] == GUARD).all(), off


def test_pfsp_expand_device_on_caller_stream():
    """children at offsets 0 and 8 (4 is refused), on the caller's stream; a chunk whose leaves lower best = 2^63-1
    takes the sequential slow path, which must write the children and lower *best on that stream as well.  The
    children array has the room the header asks for (count * jobs nodes), guarded after it; the slow path leaves the
    launch-value children of its first pass in that room, the fast path writes nothing past its children."""
    import torch
    n = 3000
    rng = np.random.default_rng(18)
    with tsb200.PfspEvaluator(14, M=n) as ev:
        t = copy_tables(ev.tables, po.Tables)
        plain = rand_pfsp(rng, 20, n)
        plain["depth"] = np.minimum(plain["depth"], 18)
        plain["limit1"] = plain["depth"] - 1
        leafy = rand_pfsp(rng, 20, n)
        leafy["depth"][::7] = 19
        leafy["limit1"] = leafy["depth"] - 1
        ev.expand(plain[:100], "lb1", 1377)  # (the host entry point first: the handle's own children buffer exists)
        for nodes, best, slow in ((plain, INT_MAX, False), (leafy, CHAPEL_MAX, True)):
            kids, sol, best_after = po.pfsp_expand(t, 1, nodes.view(po.PFSP_NODE_DTYPE), best)
            kb = kids.tobytes()
            assert (best_after < best) == slow and len(kb) > 0
            room = n * 20 * 88
            for off in (0, 8):
                s = torch.cuda.Stream()
                x, key, d_par = device_parents(torch, nodes, rand_pfsp(rng, 20, n))
                d_kids = torch.full((room + 16 + 64,), GUARD, dtype=torch.uint8, device="cuda:0")
                torch.cuda.synchronize()
                slow0 = ev.slow_rounds
                with torch.cuda.stream(s):
                    torch.cuda._sleep(SLEEP)
                    torch.bitwise_xor(x, key, out=d_par)
                    nc, ns, b = ev.expand_device("lb1", d_par.data_ptr(), n, best, d_kids.data_ptr() + off, s.cuda_stream)
                    got = d_kids.cpu().numpy()
                assert (nc, ns, b) == (kids.shape[0], sol, best_after), off
                assert ev.slow_rounds - slow0 == int(slow)
                assert got[off:off + len(kb)].tobytes() == kb, off
                assert (got[:off] == GUARD).all() and (got[off + room:] == GUARD).all(), off
                if not slow:
                    assert (got[off + len(kb):] == GUARD).all(), off
        d_par = torch.from_numpy(plain.view(np.uint8).copy()).to("cuda:0")
        d_kids = torch.empty(n * 20 * 88 + 64, dtype=torch.uint8, device="cuda:0")
        with pytest.raises(tsb200.TsbError) as e:
            ev.expand_device("lb1", d_par.data_ptr(), n, 1377, d_kids.data_ptr() + 4)
        assert e.value.code == -5  # TSB_EALIGN: children must be 8-byte aligned

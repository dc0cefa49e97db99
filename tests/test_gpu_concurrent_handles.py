"""Distinct handles driven at the same time from several host threads on one GPU, against values computed before the
threads start (the oracle, the host model of the pool, tests/golden/counts.json).

include/tsb200.h promises that distinct handles are fully concurrent and that a handle is not re-entrant; the Chapel
multi-GPU drivers rely on it (one handle per task inside `coforall gpuID`, tasks on shared OS worker threads, several
tasks per device when there are fewer GPUs than tasks).  What the handles share is exercised here from several
threads at once: cooperative persistent launches of different handles on one device, device-synchronising runtime
calls (arena growth and compaction, handle creation and destruction, host registration) while other handles are
mid-round, pinned result records of short-lived handles, process-wide page-locking behind per-handle registries,
the search drivers' handle cache and the thread-local error text.

The harness at the top runs one job per thread (`run_concurrently`): a barrier releases all jobs into their first
library call together, every library call is timed, and the run fails unless every lane (a thread, or a handle
served by several threads) made a call that overlapped another lane's call, and no two calls on one lane overlapped.
Jobs that must meet (a steal between handles owned by two threads) yield a `Meet` at fixed points of their scripts,
so that what every call returns is deterministic.  Each job appends what it got to its own list of records; the
test compares the lists after the join with lists computed before the threads started.  Every scenario also runs
once more with all its jobs in one thread (`run_serially`, the meets resolved in script order) and must give the
same records, including the transfer routes (`last_xfer`) — so the concurrent comparison is not vacuous and no
result depends on the interleaving.  The harness has CPU tests of its own (fake calls built on time.sleep)."""
import collections
import contextlib
import ctypes as C
import hashlib
import inspect
import json
import mmap
import os
import queue
import re
import threading
import time

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po
from oracle import pyoracle50 as po50
from test_gpu_host_routes import FILL, Guarded, route_of
from test_gpu_host_routes import rand_pfsp as rand_pfsp_dtype
from test_gpu_parity import copy_tables, rand_nq, rand_pfsp
from test_gpu_pool_ops import INT64_MAX, OPT14, PFR_MAX_M, ModelPool, NqProblem, PfspProblem, nq_one_pool_capacity
from test_gpu_searches import pools_wanted

PAGE = mmap.PAGESIZE
INT_MAX = 2**31 - 1
AUTO, MEMCPY, ZEROCOPY = tsb200.XFER_AUTO, tsb200.XFER_MEMCPY, tsb200.XFER_ZEROCOPY
R_ZC, R_IN, R_OUT = tsb200.XFER_ROUTE_ZEROCOPY, tsb200.XFER_ROUTE_IN_STAGED, tsb200.XFER_ROUTE_OUT_STAGED
R_PIPE = tsb200.XFER_ROUTE_PIPELINED
EINVAL, ECUDA = tsb200._lib.EINVAL, tsb200._lib.ECUDA
TIMEOUT = 600  # seconds one scenario's threads get before the run counts as hung
M_SMALL = 25


# ================================================================================================== the harness
class Meet:
    """a fixed point at which `parties` jobs meet: all arrive, one of them runs fn(ctx) while the others wait at the
    barrier (so no other party's handle is in use: the barrier alone makes fn exclusive), all leave together.  fn's
    return value is kept in `result`."""

    def __init__(self, parties, fn=None):
        self.parties, self.fn = parties, fn
        self.result = None
        self.barrier = threading.Barrier(parties)


class Ctx:
    """what a job gets: `call` times one library call on the job's lane, `record` keeps one result"""

    def __init__(self, run, lane):
        self.run, self.lane = run, lane
        self.records = []
        self.started = False

    def begin(self):
        if not self.started:
            self.started = True
            if self.run.start is not None:
                self.run.start.wait(self.run.timeout)

    def call(self, fn, *args):
        self.begin()
        t0 = time.perf_counter()
        try:
            return fn(*args)
        finally:
            self.run.log(self.lane, t0, time.perf_counter())

    def record(self, *item):
        self.records.append(norm(item))


def norm(x):
    """a record as it is kept: byte strings longer than 256 bytes by their SHA-256"""
    if isinstance(x, bytes) and len(x) > 256:
        return "sha256:" + hashlib.sha256(x).hexdigest()
    if isinstance(x, (tuple, list)):
        return type(x)(norm(v) for v in x)
    return x


class Run:
    def __init__(self, n, concurrent, timeout=TIMEOUT):
        self.timeout = timeout
        self.start = threading.Barrier(n) if concurrent and n > 1 else None
        self.ctxs = [Ctx(self, i) for i in range(n)]
        self.calls = []  # (lane, t0, t1)
        self.meets = []
        self.mu = threading.Lock()
        self.aborted = False
        self.wall = 0.0

    def log(self, lane, t0, t1):
        with self.mu:
            self.calls.append((lane, t0, t1))

    def abort(self):
        with self.mu:
            self.aborted = True
            barriers = [m.barrier for m in self.meets] + ([self.start] if self.start else [])
        for b in barriers:
            b.abort()

    def meet(self, ctx, m):
        ctx.begin()
        with self.mu:
            self.meets.append(m)
            if self.aborted:
                m.barrier.abort()
        if m.barrier.wait(self.timeout) == 0 and m.fn is not None:
            m.result = m.fn(ctx)
        m.barrier.wait(self.timeout)

    @property
    def records(self):
        return [c.records for c in self.ctxs]


def _drive(run, i, job):
    ctx = run.ctxs[i]
    r = job(ctx)
    if inspect.isgenerator(r):
        for m in r:
            run.meet(ctx, m)
    ctx.begin()  # (a job that made no call still releases the others)


def run_concurrently(jobs, timeout=TIMEOUT):
    """one thread per job, released together into their first library call; fails if a thread raised or is still
    running after `timeout` seconds (the threads are daemons: a hung one cannot keep the suite from ending)"""
    run = Run(len(jobs), True, timeout)
    errors = [None] * len(jobs)

    def body(i):
        try:
            _drive(run, i, jobs[i])
        except BaseException as e:  # noqa: BLE001 (re-raised by the joining thread)
            errors[i] = e
            run.abort()

    threads = [threading.Thread(target=body, args=(i,), name=f"job{i}", daemon=True) for i in range(len(jobs))]
    t0 = time.monotonic()
    for t in threads:
        t.start()
    for t in threads:
        t.join(max(0.0, t0 + timeout - time.monotonic()))
    run.wall = time.monotonic() - t0
    alive = [t.name for t in threads if t.is_alive()]
    if alive:
        run.abort()
        raise AssertionError(f"still running after {timeout} s: {alive}")
    failed = [(i, e) for i, e in enumerate(errors) if e is not None]
    if failed:
        # the first error that is not another thread's broken barrier is the cause
        i, e = next(((i, e) for i, e in failed if not isinstance(e, threading.BrokenBarrierError)), failed[0])
        e.add_note(f"in job {i}; jobs that failed: {[j for j, _ in failed]}")
        raise e
    return run


def run_serially(jobs):
    """the same jobs in the calling thread: plain jobs one after the other, then the generator jobs round-robin, each
    up to its next meet; a meet runs once all its parties have arrived"""
    run = Run(len(jobs), False)
    t0 = time.monotonic()
    gens = {}
    for i, job in enumerate(jobs):
        r = job(run.ctxs[i])
        if inspect.isgenerator(r):
            gens[i] = r
    waiting = {}
    while gens:
        moved = False
        for i in list(gens):
            if i in waiting:
                continue
            try:
                waiting[i] = next(gens[i])
            except StopIteration:
                del gens[i]
            moved = True
        for m in {id(m): m for m in waiting.values()}.values():
            who = [i for i, w in waiting.items() if w is m]
            if len(who) == m.parties:
                if m.fn is not None:
                    m.result = m.fn(run.ctxs[who[-1]])
                for i in who:
                    del waiting[i]
                moved = True
        assert moved, f"jobs {sorted(waiting)} wait at meets that never fill"
    run.wall = time.monotonic() - t0
    return run


def overlaps(calls):
    """(pairs of calls on different lanes whose intervals overlap, lanes without such a call, pairs of calls on one
    lane that overlap)"""
    if not calls:
        return 0, set(), 0
    lane = np.array([c[0] for c in calls])
    t0 = np.array([c[1] for c in calls])
    t1 = np.array([c[2] for c in calls])
    pairs = same = 0
    hit = np.zeros(len(calls), dtype=bool)
    for k in range(len(calls)):
        ov = (t0[k + 1:] < t1[k]) & (t0[k] < t1[k + 1:])
        other = ov & (lane[k + 1:] != lane[k])
        pairs += int(other.sum())
        same += int((ov & ~other).sum())
        if other.any():
            hit[k] = True
            hit[k + 1:][other] = True
    return pairs, set(lane.tolist()) - set(lane[hit].tolist()), same


def check_overlap(run, name=""):
    """every lane made a call that was in flight together with another lane's call; no lane had two calls in flight
    at once (a handle is not re-entrant).  Returns the number of overlapping pairs."""
    pairs, idle, same = overlaps(run.calls)
    assert same == 0, f"{name}: {same} pairs of calls on one lane overlapped"
    assert not idle, f"{name}: lanes {sorted(idle)} made no call that overlapped another lane's call"
    print(f"[concurrent] {name}: {pairs} overlapping call pairs, {len(run.calls)} calls on {len(run.ctxs)} lanes, "
          f"{run.wall:.2f} s")
    return pairs


def assert_records(got, want, name):
    """per lane: the same records in the same order (the first difference is named)"""
    assert len(got) == len(want)
    for lane, (g, w) in enumerate(zip(got, want)):
        for k, (a, b) in enumerate(zip(g, w)):
            assert a == b, f"{name}: lane {lane}, record {k} ({b[0] if b else ''}) differs"
        assert len(g) == len(w), f"{name}: lane {lane}: {len(g)} records, {len(w)} expected"


def check_scenario(name, make_jobs, want, around=None):
    """the jobs once on threads of their own (inside the context manager `around`, if any) and once in one thread,
    both against `want` (records per lane)"""
    want = norm(want)
    with around or contextlib.nullcontext():
        run = run_concurrently(make_jobs())
    assert_records(run.records, want, f"{name} (concurrent)")
    pairs = check_overlap(run, name)
    serial = run_serially(make_jobs())
    assert_records(serial.records, want, f"{name} (serial)")
    assert overlaps(serial.calls)[0] == 0
    return pairs


def check_scripts(name, scripts):
    """check_scenario for (job, want) pairs whose jobs keep no state between runs"""
    check_scenario(name, lambda: [j for j, _ in scripts], [w for _, w in scripts])


# ------------------------------------------------------------------------------------------ the harness's own tests
def sleeper(seconds, calls=3):
    def job(ctx):
        for k in range(calls):
            ctx.call(time.sleep, seconds)
            ctx.record("slept", k)
    return job


def test_harness_overlapping_fake_calls():
    run = run_concurrently([sleeper(0.05) for _ in range(4)], timeout=30)
    assert run.records == [[("slept", k) for k in range(3)]] * 4
    assert check_overlap(run, "fake") >= 4 * 3 // 2


def test_harness_serialised_job_fails_the_overlap_check():
    """the second job starts its calls only after the first has made all of its calls"""
    done = threading.Event()

    def first(ctx):
        for _ in range(3):
            ctx.call(time.sleep, 0.02)
        done.set()

    def second(ctx):
        ctx.begin()
        assert done.wait(30)
        for _ in range(3):
            ctx.call(time.sleep, 0.02)

    run = run_concurrently([first, second], timeout=30)
    with pytest.raises(AssertionError, match="made no call that overlapped"):
        check_overlap(run, "serialised")


def test_harness_reentrant_lane_fails_the_overlap_check():
    run = Run(2, False)
    run.calls = [(0, 0.0, 1.0), (0, 0.5, 1.5), (1, 0.2, 0.3)]
    with pytest.raises(AssertionError, match="on one lane overlapped"):
        check_overlap(run, "re-entrant")


def test_harness_hung_job_fails_the_timeout():
    release = threading.Event()

    def hung(ctx):
        ctx.call(release.wait)  # never set while the run is watched

    t0 = time.monotonic()
    try:
        with pytest.raises(AssertionError, match="still running after"):
            run_concurrently([sleeper(0.01), hung], timeout=1.0)
        assert time.monotonic() - t0 < 10
    finally:
        release.set()  # let the thread end


def test_harness_error_in_a_job_is_raised():
    def bad(ctx):
        ctx.call(time.sleep, 0.01)
        raise ValueError("job failed")

    def waits(ctx):
        ctx.call(time.sleep, 0.01)
        yield Meet(2)  # (never filled: `bad` is gone; the broken barrier ends this job)

    with pytest.raises(ValueError, match="job failed"):
        run_concurrently([bad, waits], timeout=30)


def test_harness_meets_are_deterministic():
    """a transfer between two jobs' state at fixed points gives the same records on threads and in one thread"""
    def make():
        state = [[0], [100]]
        meets = [Meet(2, lambda ctx, k=k: state[k % 2].append(state[1 - k % 2].pop())) for k in range(3)]

        def job(i):
            def run(ctx):
                for k in range(3):
                    ctx.call(time.sleep, 0.002 * (1 + i))
                    state[i].append(10 * i + k)
                    yield meets[k]
                    ctx.record(k, list(state[i]))
            return run
        return [job(0), job(1)]

    a = run_concurrently(make(), timeout=30)
    b = run_serially(make())
    assert a.records == b.records and len(a.records[0]) == 3


# ================================================================================================== scenarios
pytest_gpu = pytest.mark.gpu


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    """no switch of the library leaks in from the caller's environment"""
    for v in ("TSB200_NO_HANDLE_CACHE", "TSB200_NO_LB2U", "TSB200_NO_NUMA", "TSB200_NO_REGISTER", "TSB200_NO_ROUNDS",
              "TSB200_NO_SIMD16", "TSB200_NO_STEAL", "TSB200_NQ_TILE_THREADS", "TSB200_PIPE_CHUNK", "TSB200_PIPE_MIN",
              "TSB200_POOLS", "TSB200_POOL_CAP", "TSB200_ROUNDS_PROF", "TSB200_TRACE", "TSB200_XFER"):
        monkeypatch.delenv(v, raising=False)


@pytest.fixture(scope="module")
def sms():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"
    n = int(tsb200.lib().tsb_device_sm_count(0))
    assert n > 0
    return n


def masked(out, live, count):
    return np.where(live[:count], out[:count], 0).astype(out.dtype).tobytes()


class EvalSpec:
    """one handle's host-buffer evaluate and its oracle on M parents: make() creates the handle, call(ev, pin, n,
    out) runs tsb_*_evaluate on raw pointers, device(ev, d_par, n, d_out, stream) the device-resident form"""

    def __init__(self, name, M, seed, nq=None, inst=None, lb=None, best=None):
        rng = np.random.default_rng(seed)
        self.name, self.M = name, M
        if nq is not None:
            N = nq
            self.parents = rand_nq(rng, N, M)
            pv = self.parents.view(po.NQ_NODE_DTYPE)
            self.want = po.nq_evaluate(pv, N).reshape(M, N)
            self.live = po.nq_live_mask(pv, N)
            self.width, self.out_dtype = N, np.uint8
            self.make = lambda: tsb200.NQueensEvaluator(N, M=M)
            self.call = lambda ev, p, n, o: tsb200.lib().tsb_nq_evaluate(ev._h, p, n, o)
            self.device = lambda ev, p, n, o, s: ev.evaluate_device(p, n, o, s)
        else:
            kind = tsb200.LB_NAMES[lb]
            wide = tsb200.lib().tsb_taillard_nb_jobs(inst) > 20
            t = tsb200.taillard_tables50(inst) if wide else tsb200.taillard_tables(inst)
            jobs = t.jobs
            if wide:
                self.parents = rand_pfsp_dtype(rng, 50, M, tsb200.PFSP_NODE50_DTYPE)
                pv = self.parents.view(po50.PFSP_NODE_DTYPE)
                self.want = po50.pfsp_evaluate(copy_tables(t, po50.Tables), kind, pv, min(best, 2**62)).reshape(M, jobs)
                self.live = po50.pfsp_live_mask(pv, jobs)
            else:
                self.parents = rand_pfsp(rng, jobs, M)
                pv = self.parents.view(po.PFSP_NODE_DTYPE)
                self.want = po.pfsp_evaluate(copy_tables(t, po.Tables), kind, pv, best).reshape(M, jobs)
                self.live = po.pfsp_live_mask(pv, jobs)
            self.width, self.out_dtype = jobs, np.int32
            self.make = lambda: tsb200.PfspEvaluator(inst, tables=t, M=M)
            self.call = lambda ev, p, n, o: tsb200.lib().tsb_pfsp_evaluate(ev._h, kind, p, n, int(best), o)
            self.device = lambda ev, p, n, o, s: ev.evaluate_device(lb, p, n, best, o, s)


# ------------------------------------------------------------------------------------------ 1. evaluate, every route
PIPE_CHUNK, EVAL_M = 1024, 4096
NQ_TILE, NQ_SMALL = 512, 128  # csrc/nq_kernel.cuh: parents per tile of the TMA kernel, per CTA of the small one


def nq_tma_from(sms):
    """launch_nq_n: chunks of at least two 512-parent tiles per SM take the TMA-pipelined kernel, smaller ones the
    one-parent-per-thread kernel"""
    return 2 * sms * NQ_TILE


def launch_sizes(route, n):
    """the parents of each kernel launch of one host-buffer evaluate call: sub-chunks of PIPE_CHUNK when pipelined"""
    if route & R_PIPE:
        return [min(PIPE_CHUNK, n - off) for off in range(0, n, PIPE_CHUNK)]
    return [n]


def eval_script(spec, tile, extra=()):
    """(job, want, launch sizes): registered arrays in AUTO / MEMCPY / ZEROCOPY, unregistered ones, counts 1,
    tile - 1 .. tile + 1, two pipelined sizes, `extra` and M_max, then evaluate_device on a stream the thread creates
    (tile + 1, `extra`, M_max); every call's route and number of kernel launches are part of its record"""
    counts = (1, tile - 1, tile, tile + 1, PIPE_CHUNK + 1, 2 * PIPE_CHUNK + 1) + tuple(extra) + (spec.M,)
    plan = [(reg, mode, n) for reg, mode in ((True, AUTO), (True, MEMCPY), (True, ZEROCOPY), (False, AUTO))
            for n in counts]
    want, sizes = [], []
    for reg, mode, n in plan:
        route = route_of(mode, reg, reg, True, n)
        sizes += launch_sizes(route, n)
        want.append((f"{spec.name} reg={reg} mode={mode} n={n}", 0, route, len(launch_sizes(route, n)), True,
                     masked(spec.want, spec.live, n)))
    dev_counts = (tile + 1,) + tuple(extra) + (spec.M,)
    sizes += dev_counts
    want += [(f"{spec.name} device n={n}", 1, masked(spec.want, spec.live, n)) for n in dev_counts]

    def job(ctx):
        import torch
        ev = ctx.call(spec.make)
        try:
            bufs = {}
            for reg in (True, False):
                pin, out = Guarded(spec.parents.dtype, spec.M), Guarded(spec.out_dtype, spec.M * spec.width)
                pin.data[:] = spec.parents
                bufs[reg] = (pin, out)
            pin, out = bufs[True]
            ctx.call(ev.register_host, pin.span)
            ctx.call(ev.register_host, out.span)
            for reg, mode, n in plan:
                pin, out = bufs[reg]
                ctx.call(ev.set_xfer, mode)
                out.bytes[:] = FILL
                l0 = ev.kernel_launches
                rc = ctx.call(spec.call, ev, pin.ptr, n, out.ptr)
                clean = bool(out.guards_ok() and (out.bytes[n * spec.width * out.dtype.itemsize:] == FILL).all()
                             and np.array_equal(pin.data, spec.parents))
                got = out.data[: n * spec.width].reshape(n, spec.width)
                ctx.record(f"{spec.name} reg={reg} mode={mode} n={n}", rc, ctx.call(lambda: ev.last_xfer),
                           ev.kernel_launches - l0, clean, masked(got, spec.live, n))
            ctx.call(ev.unregister_host, bufs[True][0].span)
            ctx.call(ev.unregister_host, bufs[True][1].span)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                d_par = torch.from_numpy(spec.parents.view(np.uint8).copy()).to("cuda:0")
                for n in dev_counts:
                    d_out = torch.zeros(spec.M * spec.width, dtype=getattr(torch, np.dtype(spec.out_dtype).name),
                                        device="cuda:0")
                    l0 = ev.kernel_launches
                    ctx.call(spec.device, ev, d_par.data_ptr(), n, d_out.data_ptr(), s.cuda_stream)
                    got = d_out.cpu().numpy()[: n * spec.width].reshape(n, spec.width)
                    ctx.record(f"{spec.name} device n={n}", ev.kernel_launches - l0, masked(got, spec.live, n))
            s.synchronize()
        finally:
            ctx.call(ev.close)
    return job, want, sizes


def kernel_counts(prof, pattern):
    """launches per kernel whose name matches `pattern` (one group: the kernel) in a torch.profiler trace"""
    got = collections.Counter()
    for e in prof.events():
        m = re.search(pattern, e.name)
        if m:
            got[m.group(1)] += 1
    return got


@pytest_gpu
def test_evaluate_every_route_eight_threads(sms, monkeypatch):
    """8 threads, one handle each: N-Queens N = 4 (chunks below the TMA kernel's threshold: the small kernel only), 17
    and 20 (M_max two tiles past the threshold: both kernels, the TMA-pipelined one on counts from the threshold up,
    zero-copy on the caller's registered arrays and on device arrays); PFSP ta001 lb2 at INT_MAX, ta014 lb1, ta021
    lb1_d, ta020 lb2 at its optimum; a 50-job handle (ta031 lb1).  Handles made with TSB200_PIPE_MIN=1,
    TSB200_PIPE_CHUNK=1024 (a pipelined call launches one kernel per 1024 parents).  A torch.profiler trace of the
    concurrent run counts the launches of each N-Queens evaluate kernel."""
    import torch
    monkeypatch.setenv("TSB200_PIPE_MIN", "1")
    monkeypatch.setenv("TSB200_PIPE_CHUNK", str(PIPE_CHUNK))
    opt = lambda inst: int(tsb200.lib().tsb_taillard_best_ub(inst))  # noqa: E731
    T = nq_tma_from(sms)
    big = (T - 1, T, T + NQ_TILE - 1, T + NQ_TILE, T + NQ_TILE + 1)  # the threshold and the TMA kernel's tile edges
    M_big = T + 2 * NQ_TILE
    nq = [("nq4", 4, EVAL_M, ()), ("nq17", 17, M_big, big), ("nq20", 20, M_big, big)]
    scripts = [eval_script(EvalSpec(name, M, 1 + k, nq=N), NQ_SMALL, extra) for k, (name, N, M, extra) in enumerate(nq)]
    scripts += [eval_script(s, tile)[:2] + (None,) for s, tile in (
        (EvalSpec("ta001 lb2", EVAL_M, 4, inst=1, lb="lb2", best=INT_MAX), 64),
        (EvalSpec("ta014 lb1", EVAL_M, 5, inst=14, lb="lb1", best=opt(14)), 128),
        (EvalSpec("ta021 lb1_d", EVAL_M, 6, inst=21, lb="lb1_d", best=opt(21)), 128),
        (EvalSpec("ta020 lb2", EVAL_M, 7, inst=20, lb="lb2", best=opt(20)), 64),
        (EvalSpec("ta031 lb1", EVAL_M, 8, inst=31, lb="lb1", best=opt(31)), 64))]
    want_kernels = collections.Counter()
    for (_, N, _, _), (_, _, sizes) in zip(nq, scripts):
        for n in sizes:
            want_kernels[f"nq_evaluate_{'' if n >= T else 'small_'}kernel<{N}>"] += 1
    assert want_kernels["nq_evaluate_kernel<17>"] >= 10 and "nq_evaluate_kernel<4>" not in want_kernels
    prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA],
                                  acc_events=True)
    check_scenario("1 evaluate", lambda: [j for j, _, _ in scripts], [w for _, w, _ in scripts], around=prof)
    assert kernel_counts(prof, r"(nq_evaluate_(?:small_)?kernel<\d+>)") == want_kernels


# ------------------------------------------------------------------------------------------ 2. fused expand
def nq_expand_script(N, chunks, on_device):
    want = []
    for k, ch in enumerate(chunks):
        kids, sol = po.nq_expand(ch.view(po.NQ_NODE_DTYPE), N)
        want.append((f"nq{N} chunk {k}", kids.shape[0], sol, kids.tobytes()))

    def job(ctx):
        import torch
        ev = ctx.call(tsb200.NQueensEvaluator, N, 1, max(c.shape[0] for c in chunks))
        try:
            s = torch.cuda.Stream()
            for k, ch in enumerate(chunks):
                if on_device:
                    with torch.cuda.stream(s):
                        d_par = torch.from_numpy(ch.view(np.uint8).copy()).to("cuda:0")
                        d_kids = torch.zeros(ch.shape[0] * N * 21 + 16, dtype=torch.uint8, device="cuda:0")
                        nc, ns = ctx.call(ev.expand_device, d_par.data_ptr(), ch.shape[0], d_kids.data_ptr(), s.cuda_stream)
                        kb = d_kids[: nc * 21].cpu().numpy().tobytes()
                else:
                    kids, ns = ctx.call(ev.expand, ch)
                    nc, kb = kids.shape[0], kids.tobytes()
                ctx.record(f"nq{N} chunk {k}", nc, ns, kb)
        finally:
            ctx.call(ev.close)
    return job, want


def pfsp_expand_script(lb, chunks, on_device):
    """chunks: (parents, best); a chunk in which a leaf lowers best goes through the sequential rule (slow_rounds)"""
    t = tsb200.taillard_tables(14)
    to = copy_tables(t, po.Tables)
    kind = tsb200.LB_NAMES[lb]
    want = []
    for k, (ch, best) in enumerate(chunks):
        kids, sol, after = po.pfsp_expand(to, kind, ch.view(po.PFSP_NODE_DTYPE), best)
        want.append((f"{lb} chunk {k}", kids.shape[0], sol, after, int(after < best), kids.tobytes()))
    assert any(w[4] for w in want) and not all(w[4] for w in want)

    def job(ctx):
        import torch
        ev = ctx.call(lambda: tsb200.PfspEvaluator(14, tables=t, M=max(c.shape[0] for c, _ in chunks)))
        try:
            s = torch.cuda.Stream()
            for k, (ch, best) in enumerate(chunks):
                slow0 = ev.slow_rounds
                if on_device:
                    with torch.cuda.stream(s):
                        d_par = torch.from_numpy(ch.view(np.uint8).copy()).to("cuda:0")
                        d_kids = torch.zeros(ch.shape[0] * 20 * 88, dtype=torch.uint8, device="cuda:0")
                        nc, ns, after = ctx.call(ev.expand_device, lb, d_par.data_ptr(), ch.shape[0], best,
                                                 d_kids.data_ptr(), s.cuda_stream)
                        kb = d_kids[: nc * 88].cpu().numpy().tobytes()
                else:
                    kids, ns, after = ctx.call(ev.expand, ch, lb, best)
                    nc, kb = kids.shape[0], kids.tobytes()
                ctx.record(f"{lb} chunk {k}", nc, ns, after, ev.slow_rounds - slow0, kb)
        finally:
            ctx.call(ev.close)
    return job, want


def pfsp_chunks(rng, count):
    plain = rand_pfsp(rng, 20, count)
    plain["depth"] = np.minimum(plain["depth"], 18)  # no leaves: best stays
    plain["limit1"] = plain["depth"] - 1
    leafy = rand_pfsp(rng, 20, count)
    leafy["depth"][::7] = 19  # leaves: a chunk at best = 2^63 - 1 lowers it
    leafy["limit1"] = leafy["depth"] - 1
    return [(plain, OPT14), (leafy, INT64_MAX), (plain, INT64_MAX), (leafy, OPT14)]


@pytest_gpu
def test_expand_six_threads(sms):
    """N-Queens expand (N = 14) and expand_device (N = 17, on the thread's stream); PFSP expand for lb1, lb1_d and
    lb2 and expand_device for lb1, with chunks in which a leaf lowers best: children byte for byte, best, slow_rounds"""
    rng = np.random.default_rng(20)
    nq14 = [rand_nq(rng, 14, n, depth_lo=4) for n in (3000, 1, 5000) * 4]
    nq17 = [rand_nq(rng, 17, n, depth_lo=8) for n in (4000, 2, 3000) * 4]
    pf = {lb: pfsp_chunks(rng, 2500) * 3 for lb in ("lb1", "lb1_d", "lb2", "dev")}
    check_scripts("2 expand", [nq_expand_script(14, nq14, False), nq_expand_script(17, nq17, True),
                               pfsp_expand_script("lb1", pf["lb1"], False), pfsp_expand_script("lb1_d", pf["lb1_d"], False),
                               pfsp_expand_script("lb2", pf["lb2"], False), pfsp_expand_script("lb1", pf["dev"], True)])


# ------------------------------------------------------------------------------------------ 3. device pools
class PoolLane:
    """one pool's script on a device handle (ev) or on the host model (ev None): each op records what it returned
    and the pool size after it"""

    def __init__(self, prob, ev=None):
        self.prob, self.ev = prob, ev
        self.model = ModelPool(prob) if ev is None else None
        self.best = prob.best0

    def apply(self, ctx, op):
        kind, args = op[0], op[1:]
        ev, mod, prob = self.ev, self.model, self.prob
        if kind == "push":
            if ev:
                ctx.call(ev.pool_push, args[0])
            else:
                mod.push(args[0])
            got = None
        elif kind == "step":
            m, M = args
            if ev:
                got, self.best = ctx.call(prob.step, ev, m, M, self.best)
            else:
                got = mod.step(m, M)
                self.best = mod.best
        elif kind == "run":
            m, M, k = args
            if ev:
                got, self.best = ctx.call(prob.run, ev, m, M, self.best, k)
            else:
                got = mod.run(m, M, k)
                self.best = mod.best
        else:  # drain, and push the nodes back
            if ev:
                nodes = ctx.call(ev.pool_drain)
                if nodes.shape[0]:
                    ctx.call(ev.pool_push, nodes)
            else:
                nodes = mod.drain()
                mod.push(nodes)
            got = np.ascontiguousarray(nodes).tobytes()
        ctx.record(kind, args[0].shape[0] if kind == "push" else args, tuple(got) if isinstance(got, tuple) else got,
                   self.best, self.size(ctx))

    def size(self, ctx):
        return ctx.call(lambda: self.ev.pool_size) if self.ev else self.model.size

    def steal_from(self, ctx, victim, m):
        if self.ev:
            return ctx.call(self.ev.pool_steal_from, victim.ev, m)
        return victim.model.steal_to(self.model, m)


def pool_ops(prob, rng, n_ops, inside, outside):
    ops = [("push", prob.nodes(rng, 3001))]
    for _ in range(n_ops - 1):
        op = rng.choice(["push", "step", "run", "run", "run", "drain"])
        if op == "push":
            ops.append(("push", prob.nodes(rng, int(rng.choice([1, 37, 3001])))))
        elif op == "step":
            ops.append(("step", int(rng.choice([1, 25])), int(rng.choice([300, 5000]))))
        elif op == "run":
            ops.append(("run", int(rng.choice([1, 25])), int(rng.choice([inside, inside, outside])),
                        int(rng.integers(1, 4))))
        else:
            ops.append(("drain",))
    ops += [("run", 25, inside, 2), ("drain",)]
    return ops


class PoolScenario:
    """lanes of pool scripts, steals at fixed points between pairs of lanes, and multi-pool lanes; the expected
    records are the same scripts run on the host model by run_serially"""

    def __init__(self, lanes, steals, multi):
        self.lanes = lanes    # [(problem, make_handle, ops)]
        self.steals = steals  # {(victim, thief): [(after op index, m)]}
        self.multi = multi    # [(kind, problems, pushes, rounds)]

    def jobs(self, on_device):
        objs, ctx_of, meets = {}, {}, {}
        for (v, t), points in self.steals.items():
            for k, m in points:
                def fn(ctx, v=v, t=t, m=m):  # (the thief's thread waits at the meet: its records stay in order)
                    got = objs[t].steal_from(ctx, objs[v], m)
                    ctx_of[t].record("steal", v, got)
                    return got
                meets.setdefault(v, {})[k] = meets.setdefault(t, {})[k] = Meet(2, fn)

        def single(i, prob, make, ops):
            def job(ctx):
                ctx_of[i] = ctx
                ev = ctx.call(make) if on_device else None
                try:
                    objs[i] = PoolLane(prob, ev)
                    for k, op in enumerate(ops):
                        objs[i].apply(ctx, op)
                        if k in meets.get(i, {}):
                            yield meets[i][k]
                finally:
                    if ev is not None:
                        ctx.call(ev.close)
            return job

        def multi(kind, probs, pushes, rounds):
            def job(ctx):
                lanes, evs, owner = [], [], None
                if on_device:
                    owner = ctx.call(probs[0].handle, 5000)
                    evs = [owner] + [sibling(ctx, owner, kind, i) for i in range(1, len(probs))]
                try:
                    lanes = [PoolLane(p, evs[i] if evs else None) for i, p in enumerate(probs)]
                    for r, (nodes, k) in enumerate(zip(pushes, rounds)):
                        for lane, nd in zip(lanes, nodes):
                            lane.apply(ctx, ("push", nd))
                        if on_device:
                            if kind == "nq":
                                got = ctx.call(tsb200.nqueens_pool_run_multi, evs, 1, 5000, k)
                            else:
                                got = ctx.call(tsb200.pfsp_pool_run_multi, evs, "lb1", 1, 5000,
                                               [ln.best for ln in lanes], k)
                                for ln, g in zip(lanes, got):
                                    ln.best = g[4]
                            got = [tuple(g[:4]) for g in got]
                        else:
                            got = [ln.model.run(1, 5000, k) for ln in lanes]
                            for ln in lanes:
                                ln.best = ln.model.best
                        ctx.record("multi", r, got, [ln.best for ln in lanes], [ln.size(ctx) for ln in lanes])
                        for ln in lanes:
                            ln.apply(ctx, ("drain",))
                    yield from ()
                finally:
                    if owner is not None:
                        ctx.call(owner.close)
            return job

        jobs = [single(i, p, mk, ops) for i, (p, mk, ops) in enumerate(self.lanes)]
        return jobs + [multi(*x) for x in self.multi]


class NqSibling(tsb200.NQueensEvaluator):
    """a sibling pool of an N-Queens handle: destroyed with its owner"""

    def close(self):
        self._h = C.c_void_p()

    __del__ = close


def sibling(ctx, owner, kind, i):
    if kind == "pfsp":
        return ctx.call(owner.sibling, i)
    h = C.c_void_p()
    tsb200.check(ctx.call(tsb200.lib().tsb_nq_sibling, owner._h, i, C.byref(h)), "tsb_nq_sibling")
    sib = NqSibling.__new__(NqSibling)
    sib.__dict__.update(N=owner.N, g=owner.g, M=owner.M, device=owner.device, _h=h)
    return sib


def pool_scenario(sms, seed):
    rng = np.random.default_rng(seed)
    nq_in = nq_one_pool_capacity(sms)
    lanes = []
    for N in (12, 12, 14, 15):
        prob = NqProblem(N)
        lanes.append((prob, lambda N=N: tsb200.NQueensEvaluator(N, M=nq_in + 1), pool_ops(prob, rng, 12, nq_in, nq_in + 1)))
    for lb, best in (("lb1", OPT14), ("lb1_d", INT64_MAX)):
        prob = PfspProblem(lb, best)
        lanes.append((prob, lambda: tsb200.PfspEvaluator(14, M=PFR_MAX_M + 1),
                      pool_ops(prob, rng, 12, PFR_MAX_M, PFR_MAX_M + 1)))
    steals = {(0, 1): [(4, 1)], (1, 0): [(9, 25)], (4, 5): [(3, 1), (10, 25)]}
    nq_multi = [NqProblem(12)] * 4
    pf_multi = [PfspProblem("lb1", b) for b in (OPT14, INT64_MAX, OPT14 + 40, OPT14)]
    multi = []
    for kind, probs in (("nq", nq_multi), ("pfsp", pf_multi)):
        pushes = [[p.nodes(rng, int(n)) for p, n in zip(probs, rng.choice([1, 300, 3001], size=4))] for _ in range(3)]
        multi.append((kind, probs, pushes, (1, 3, 2)))
    return PoolScenario(lanes, steals, multi)


@pytest_gpu
@pytest.mark.parametrize("cap", [None, 2000])
def test_device_pools_eight_threads(sms, cap, monkeypatch):
    """N-Queens pools (N = 12, 12, 14, 15) and PFSP ta014 pools (lb1 at the optimum, lb1_d at 2^63 - 1) running push /
    pool_step / pool_run (inside and outside the persistent kernels) / drain scripts, steals between the two N = 12
    lanes and between the PFSP lanes at fixed points, nqueens_pool_run_multi and pfsp_pool_run_multi (per-pool
    incumbents) on four pools each; with a 2000-record initial arena, growth and compaction (cudaMalloc / cudaFree)
    happen while other threads' cooperative kernels run"""
    if cap:
        monkeypatch.setenv("TSB200_POOL_CAP", str(cap))
    sc = pool_scenario(sms, 30 + (cap or 0))
    want = run_serially(sc.jobs(on_device=False)).records
    assert sum(r[0] == "steal" and r[2] > 0 for rec in want for r in rec) >= 2
    check_scenario(f"3 device pools cap={cap}", lambda: sc.jobs(on_device=True), want)


# ------------------------------------------------------------------------------------------ 4. short-lived handles
def short_lived_script(rng, count):
    """20 handles one after the other: N-Queens (register the parents, one expand, destroy) and PFSP (register,
    evaluate zero-copy, one expand, pool_push + a pool_run of a few rounds, destroy)"""
    t = tsb200.taillard_tables(14)
    to = copy_tables(t, po.Tables)
    pprob = PfspProblem("lb1", OPT14)
    steps, want = [], []
    for k in range(count):
        if k % 2 == 0:
            par = rand_nq(rng, 13, 2000, depth_lo=3)
            kids, sol = po.nq_expand(par.view(po.NQ_NODE_DTYPE), 13)
            steps.append(("nq", par))
            want.append((f"nq handle {k}", 0, kids.shape[0], sol, kids.tobytes()))
        else:
            par = rand_pfsp(rng, 20, 2000)
            par["depth"] = np.minimum(par["depth"], 18)
            par["limit1"] = par["depth"] - 1
            bounds = po.pfsp_evaluate(to, 1, par.view(po.PFSP_NODE_DTYPE), OPT14).reshape(-1, 20)
            live = po.pfsp_live_mask(par.view(po.PFSP_NODE_DTYPE), 20)
            kids, sol, after = po.pfsp_expand(to, 1, par.view(po.PFSP_NODE_DTYPE), OPT14)
            start = pprob.nodes(rng, 500)
            mod = ModelPool(pprob)
            mod.push(start)
            tot = mod.run(1, 2000, 3)
            steps.append(("pfsp", par, start))
            want.append((f"pfsp handle {k}", R_ZC, masked(bounds, live, 2000), kids.shape[0], sol, after,
                         kids.tobytes(), tot, mod.best, mod.size))

    def job(ctx):
        for k, st in enumerate(steps):
            if st[0] == "nq":
                ev = ctx.call(tsb200.NQueensEvaluator, 13, 1, 2000)
                try:
                    pin = Guarded(tsb200.NQ_NODE_DTYPE, 2000)
                    pin.data[:] = st[1]
                    ctx.call(ev.register_host, pin.span)
                    kids, ns = ctx.call(ev.expand, pin.data)
                    ctx.record(f"nq handle {k}", 0, kids.shape[0], ns, kids.tobytes())
                finally:
                    ctx.call(ev.close)
            else:
                ev = ctx.call(lambda: tsb200.PfspEvaluator(14, tables=t, M=2000))
                try:
                    pin, out = Guarded(tsb200.PFSP_NODE_DTYPE, 2000), Guarded(np.int32, 2000 * 20)
                    pin.data[:] = st[1]
                    ctx.call(ev.register_host, pin.span)
                    ctx.call(ev.register_host, out.span)
                    ctx.call(ev.evaluate_gpu, pin.data, 2000 * 20, OPT14, "lb1", out.data)
                    route = ctx.call(lambda: ev.last_xfer)
                    got = out.data.reshape(-1, 20)
                    kids, ns, after = ctx.call(ev.expand, pin.data, "lb1", OPT14)
                    ctx.call(ev.pool_push, st[2])
                    r = ctx.call(ev.pool_run, "lb1", 1, 2000, OPT14, 3)
                    ctx.record(f"pfsp handle {k}", route, masked(got, live_of(st[1]), 2000), kids.shape[0], ns, after,
                               kids.tobytes(), tuple(r[:4]), r[4], ctx.call(lambda: ev.pool_size))
                finally:
                    ctx.call(ev.close)
    return job, want


def live_of(par):
    return po.pfsp_live_mask(par.view(po.PFSP_NODE_DTYPE), 20)


def long_pool_script(prob, start, M, calls, rounds):
    mod = ModelPool(prob)
    mod.push(start)
    want = [("run", k, mod.run(1, M, rounds), mod.best, mod.size) for k in range(calls)]
    want.append(("drain", np.ascontiguousarray(mod.drain()).tobytes()))

    def job(ctx):
        ev = ctx.call(prob.handle, M)
        try:
            ctx.call(ev.pool_push, start)
            best = prob.best0
            for k in range(calls):
                got, best = ctx.call(prob.run, ev, 1, M, best, rounds)
                ctx.record("run", k, tuple(got), best, ctx.call(lambda: ev.pool_size))
            ctx.record("drain", ctx.call(ev.pool_drain).tobytes())
        finally:
            ctx.call(ev.close)
    return job, want


@pytest_gpu
def test_short_lived_handles_beside_long_running_ones(sms):
    """one thread creates, uses and destroys 20 handles while two threads run long pool_run scripts: every
    short-lived handle's first expand and first pool_run reads its own freshly allocated pinned result records"""
    rng = np.random.default_rng(40)
    nq15 = NqProblem(15)
    pf = PfspProblem("lb1", OPT14)
    nq_start, pf_start = rand_nq(rng, 15, 2000, depth_lo=4, depth_hi=5), pf.nodes(rng, 3000)  # (neither runs dry)
    check_scripts("4 short-lived handles", [short_lived_script(rng, 20), long_pool_script(nq15, nq_start, 20000, 60, 2),
                                            long_pool_script(pf, pf_start, 5000, 60, 2)])


# ------------------------------------------------------------------------------------------ 5. whole searches
def search_record(st, D):
    return (st.explored_tree, st.explored_sol, st.best, list(st.per_gpu_tree[:D]), st.steals)


def nq_whole_record(st):
    """the N-Queens search with several pools per task: totals (each task's step 2 is not any oracle part's)"""
    return (st.explored_tree, st.explored_sol, st.best, st.steals, st.per_gpu_tree[0] > 0 and st.per_gpu_tree[1] > 0)


def nq_part_record(st, p):
    return (st.explored_tree, st.explored_sol, st.steals, sum(st.per_gpu_tree) == st.per_gpu_tree[p])


@pytest_gpu
def test_whole_searches_at_the_same_time(sms, golden_dir, monkeypatch):
    """nqueens_search_device(14, D = 2) with its default pools per task (the multi-pool persistent kernel), both parts
    of that split (nqueens_search_device_part), pfsp_search_device(ta014, lb1, ub = 1, D = 2) and the host-pool
    nqueens_search(13), twice each, and a thread that frees the cached handles between the searches and while the
    second ones run.  TSB200_NO_STEAL=1: the parts are the oracle's part searches (with the warm-up pool of D tasks of
    P pools, as test_gpu_searches.test_nq_parts), the PFSP tasks' trees the oracle's part trees, and the totals the
    reference's counts."""
    monkeypatch.setenv("TSB200_NO_STEAL", "1")
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))
    M, D = 50000, 2
    P = pools_wanted(sms, M)
    nq_parts = [po.nq_search_offload_part(14, 1, M_SMALL, M, D, p, D * M_SMALL * P) for p in range(D)]
    pf_tasks = [po.pfsp_search_offload_part(14, 1, 1, M_SMALL, M, D, p).task_tree[p] for p in range(D)]
    c14, c13, p14 = counts["nqueens"]["14"], counts["nqueens"]["13"], counts["pfsp"]["ta014_lb1_ub1"]
    assert sum(w.tree for w in nq_parts) == c14["tree"] and sum(w.sol for w in nq_parts) == c14["sol"]
    searches = [
        (lambda: nq_whole_record(tsb200.nqueens_search_device(14, 1, M_SMALL, M, D)),
         (c14["tree"], c14["sol"], 0, 0, True)),
        (lambda: search_record(tsb200.pfsp_search_device(14, "lb1", 1, M_SMALL, M, D), D),
         (p14["tree"], p14["sol"], p14["best"], pf_tasks, 0)),
        (lambda: search_record(tsb200.nqueens_search(13, 1, M_SMALL, M, 1), 0), (c13["tree"], c13["sol"], 0, [], 0)),
    ] + [(lambda p=p: nq_part_record(tsb200.nqueens_search_device_part(14, 1, M_SMALL, M, D, p), p),
          (w.tree, w.sol, 0, True)) for p, w in enumerate(nq_parts)]
    want = [[("search", k, w) for k in range(2)] for _, w in searches] + [[("released", 4)]]

    def jobs():
        meets = [Meet(len(searches) + 1), Meet(len(searches) + 1)]

        def searcher(run):
            def job(ctx):
                for k in range(2):
                    ctx.record("search", k, ctx.call(run))
                    yield meets[k]
            return job

        def releaser(ctx):
            n = 0
            for m in meets:
                yield m
                ctx.call(tsb200.lib().tsb_release_cached_handles)
                n += 1
                if m is meets[0]:  # and while the second searches run
                    time.sleep(0.05)
                    ctx.call(tsb200.lib().tsb_release_cached_handles)
                    n += 1
            ctx.call(tsb200.lib().tsb_release_cached_handles)
            ctx.record("released", n + 1)
        return [searcher(run) for run, _ in searches] + [releaser]

    check_scenario("5 whole searches", jobs, want)


# ------------------------------------------------------------------------------------------ 6. one handle, many threads
class Workers:
    """worker threads that take one handle's calls, call k on worker k % n: no two calls are in flight at once"""

    def __init__(self, n):
        self.qs = [queue.Queue() for _ in range(n)]
        self.used = set()
        self.threads = [threading.Thread(target=self._serve, args=(q,), daemon=True) for q in self.qs]
        for t in self.threads:
            t.start()
        self.k = 0

    def _serve(self, q):
        while True:
            item = q.get()
            if item is None:
                return
            fn, box, done = item
            try:
                box.append((True, fn()))
            except BaseException as e:  # noqa: BLE001 (re-raised by the caller)
                box.append((False, e))
            self.used.add(threading.get_ident())
            done.set()

    def __call__(self, ctx, fn, *args):
        box, done = [], threading.Event()
        self.qs[self.k % len(self.qs)].put((lambda: ctx.call(fn, *args), box, done))
        self.k += 1
        assert done.wait(TIMEOUT)
        ok, v = box[0]
        if not ok:
            raise v
        return v

    def close(self):
        for q in self.qs:
            q.put(None)
        for t in self.threads:
            t.join(TIMEOUT)


def one_handle_script(kind, seed):
    """the script of one handle whose calls move between three worker threads: evaluate on registered arrays, a
    TSB_EINVAL call, expand, pool push / run / step / drain, evaluate again"""
    rng = np.random.default_rng(seed)
    M = 3000
    if kind == "nq":
        N = 12
        par = rand_nq(rng, N, M)
        pv = par.view(po.NQ_NODE_DTYPE)
        ev_want = masked(po.nq_evaluate(pv, N).reshape(M, N), po.nq_live_mask(pv, N), M)
        chunk = rand_nq(rng, N, 1000, depth_lo=5)
        kids, sol = po.nq_expand(chunk.view(po.NQ_NODE_DTYPE), N)
        prob, width, odt = NqProblem(N), N, np.uint8
        make = lambda: tsb200.NQueensEvaluator(N, M=M)  # noqa: E731
        evaluate = lambda ev, p, o: ev.evaluate_gpu(p, M * N, o)  # noqa: E731
        bad = lambda ev, p, o: tsb200.lib().tsb_nq_evaluate(ev._h, p.ctypes.data, M + 1, o.ctypes.data)  # noqa: E731
        expand = lambda ev: ev.expand(chunk)[:2]  # noqa: E731
        exp_want = (kids.tobytes(), sol)
        live = po.nq_live_mask(pv, N)
    else:
        t = tsb200.taillard_tables(14)
        to = copy_tables(t, po.Tables)
        par = rand_pfsp(rng, 20, M)
        pv = par.view(po.PFSP_NODE_DTYPE)
        live = po.pfsp_live_mask(pv, 20)
        ev_want = masked(po.pfsp_evaluate(to, 2, pv, OPT14).reshape(M, 20), live, M)
        chunk, _ = pfsp_chunks(rng, 1000)[1]
        kids, sol, after = po.pfsp_expand(to, 0, chunk.view(po.PFSP_NODE_DTYPE), INT64_MAX)
        prob, width, odt = PfspProblem("lb1", OPT14), 20, np.int32
        make = lambda: tsb200.PfspEvaluator(14, tables=t, M=M)  # noqa: E731
        evaluate = lambda ev, p, o: ev.evaluate_gpu(p, M * 20, OPT14, "lb2", o)  # noqa: E731
        bad = lambda ev, p, o: tsb200.lib().tsb_pfsp_evaluate(ev._h, 7, p.ctypes.data, M, OPT14, o.ctypes.data)  # noqa: E731
        expand = lambda ev: ev.expand(chunk, "lb1_d", INT64_MAX)  # noqa: E731
        exp_want = (kids.tobytes(), sol, after)
    start = prob.nodes(rng, 3001)
    mod = ModelPool(prob)
    mod.push(start)
    r1 = mod.run(1, M, 2)
    s1 = mod.step(25, 300)
    best1 = mod.best
    r2 = mod.run(1, M, 2)
    drained = np.ascontiguousarray(mod.drain()).tobytes()
    want = [("evaluate", R_ZC, ev_want), ("einval", EINVAL), ("evaluate", R_ZC, ev_want), ("expand", exp_want),
            ("run", r1), ("step", s1, best1), ("run", r2, mod.best), ("drain", drained), ("workers", 3)]

    def job(ctx):
        w, ev = Workers(3), None
        try:
            ev = w(ctx, make)
            pin, out = Guarded(par.dtype, M), Guarded(odt, M * width)
            pin.data[:] = par
            w(ctx, ev.register_host, pin.span)
            w(ctx, ev.register_host, out.span)
            for k in range(2):
                out.bytes[:] = FILL
                w(ctx, evaluate, ev, pin.data, out.data)
                ctx.record("evaluate", w(ctx, lambda: ev.last_xfer), masked(out.data.reshape(M, width), live, M))
                if k == 0:
                    ctx.record("einval", w(ctx, bad, ev, pin.data, out.data))
            got = w(ctx, expand, ev)
            ctx.record("expand", (got[0].tobytes(),) + tuple(got[1:]))
            w(ctx, ev.pool_push, start)
            best = prob.best0
            got, best = w(ctx, prob.run, ev, 1, M, best, 2)
            ctx.record("run", tuple(got))
            got, best = w(ctx, prob.step, ev, 25, 300, best)
            ctx.record("step", tuple(got), best)
            got, best = w(ctx, prob.run, ev, 1, M, best, 2)
            ctx.record("run", tuple(got), best)
            ctx.record("drain", w(ctx, ev.pool_drain).tobytes())
            w(ctx, ev.unregister_host, pin.span)
            w(ctx, ev.unregister_host, out.span)
        finally:
            try:
                if ev is not None:
                    w(ctx, ev.close)
            finally:
                w.close()
        ctx.record("workers", len(w.used - {threading.get_ident()}))
    return job, want


@pytest_gpu
def test_one_handle_moving_between_worker_threads(sms):
    """an N-Queens and a PFSP handle, each served by three worker threads in turn (a Chapel task moving between
    workers): results match the oracle, a refused call leaves the handle working, the two handles overlap and no
    handle ever has two calls in flight"""
    check_scripts("6 one handle, many threads", [one_handle_script("nq", 60), one_handle_script("pfsp", 61)])


# ------------------------------------------------------------------------------------------ 7. registration
REG_LOOPS = 200


def nq_eval_record(ctx, ev, pin, out, n, N):
    """(status, route, sentinels of both arrays intact and nothing written past n * N labels, labels)"""
    out.bytes[:] = FILL
    rc = ctx.call(tsb200.lib().tsb_nq_evaluate, ev._h, pin.ptr, n, out.ptr)
    clean = bool(out.guards_ok() and (out.bytes[n * N:] == FILL).all() and pin.guards_ok())
    return rc, ctx.call(lambda: ev.last_xfer), clean, out.data[: n * N].tobytes()


@pytest_gpu
def test_one_array_registered_by_two_handles(sms):
    """handle A registers X, then handle B registers X: B gets TSB_ECUDA (the range is page-locked already; the text
    is in B's thread's tsb_last_cuda_error, A's thread's stays empty); A evaluates X zero-copy while B's calls on X
    are staged, both correct; once A has unregistered X, B can register it and evaluate zero-copy"""
    N, n = 10, 4096
    x_nodes = rand_nq(np.random.default_rng(70), N, n)
    xv = x_nodes.view(po.NQ_NODE_DTYPE)
    lab = po.nq_evaluate(xv, N).reshape(n, N)
    live = po.nq_live_mask(xv, N)
    texts = []  # per run: A's thread's tsb_last_cuda_error at the end (the serial run shares B's thread)

    def jobs():
        X = Guarded(tsb200.NQ_NODE_DTYPE, n)
        texts.append([])
        X.data[:] = x_nodes
        meets = [Meet(2) for _ in range(3)]

        def run_loop(ctx, ev, out, count):
            for k in range(count):
                rc, route, clean, got = nq_eval_record(ctx, ev, X, out, n, N)
                clean = clean and np.array_equal(X.data, x_nodes)
                ctx.record("eval", rc, route, clean, masked(np.frombuffer(got, np.uint8).reshape(n, N), live, n))

        def a(ctx):
            ev = ctx.call(tsb200.NQueensEvaluator, N, 1, n)
            out = Guarded(np.uint8, n * N)
            try:
                ctx.call(ev.register_host, X.span)
                ctx.call(ev.register_host, out.span)
                yield meets[0]
                run_loop(ctx, ev, out, REG_LOOPS)
                yield meets[1]
                ctx.call(ev.unregister_host, X.span)
                yield meets[2]
                run_loop(ctx, ev, out, 5)
                ctx.call(ev.unregister_host, out.span)
                texts[-1].append(tsb200.lib().tsb_last_cuda_error())
            finally:
                ctx.call(ev.close)

        def b(ctx):
            ev = ctx.call(tsb200.NQueensEvaluator, N, 1, n)
            out = Guarded(np.uint8, n * N)
            try:
                ctx.call(ev.register_host, out.span)
                yield meets[0]
                rc = ctx.call(tsb200.lib().tsb_nq_register_host, ev._h, X.span.ctypes.data, X.span.nbytes)
                ctx.record("register X", rc, b"cudaHostRegister" in tsb200.lib().tsb_last_cuda_error())
                run_loop(ctx, ev, out, REG_LOOPS)
                yield meets[1]
                yield meets[2]
                ctx.call(ev.register_host, X.span)
                run_loop(ctx, ev, out, 5)
                ctx.call(ev.unregister_host, X.span)
                ctx.call(ev.unregister_host, out.span)
            finally:
                ctx.call(ev.close)
        return [a, b]

    ok = masked(lab, live, n)
    want = [[("eval", 0, R_ZC, True, ok)] * REG_LOOPS + [("eval", 0, R_IN, True, ok)] * 5,
            [("register X", ECUDA, True)] + [("eval", 0, R_IN, True, ok)] * REG_LOOPS + [("eval", 0, R_ZC, True, ok)] * 5]
    check_scenario("7 one array, two handles", jobs, want)
    assert texts[0] == [b""]  # B's failure did not reach A's thread


@pytest_gpu
@pytest.mark.parametrize("first", [0, 1])
def test_two_handles_register_ranges_in_one_page(sms, first):
    """an N-Queens and a PFSP handle on two threads register disjoint arrays in one page at the same time and
    evaluate on them zero-copy; the one that unregisters first goes on staged, the other stays zero-copy and correct
    until it unregisters as well"""
    rng = np.random.default_rng(71)
    N, nn, npf = 8, 16, 8
    nq_par, pf_par = rand_nq(rng, N, nn), rand_pfsp(rng, 20, npf)
    t = tsb200.taillard_tables(14)
    nqv, pfv = nq_par.view(po.NQ_NODE_DTYPE), pf_par.view(po.PFSP_NODE_DTYPE)
    want_nq = masked(po.nq_evaluate(nqv, N).reshape(nn, N), po.nq_live_mask(nqv, N), nn)
    want_pf = masked(po.pfsp_evaluate(copy_tables(t, po.Tables), 1, pfv, OPT14).reshape(npf, 20),
                     po.pfsp_live_mask(pfv, 20), npf)

    def jobs():
        raw = np.zeros(4 * PAGE, dtype=np.uint8)
        page = raw[-raw.ctypes.data % PAGE:][PAGE:2 * PAGE]
        arrays = [(page[64:64 + 21 * nn].view(tsb200.NQ_NODE_DTYPE), page[512:512 + N * nn]),
                  (page[1024:1024 + 88 * npf].view(tsb200.PFSP_NODE_DTYPE), page[2048:2048 + 80 * npf].view(np.int32))]
        arrays[0][0][:] = nq_par
        arrays[1][0][:] = pf_par
        # every byte of the buffer outside the four arrays: nothing writes there (either lane may check it any time)
        free = np.ones(raw.size, dtype=bool)
        for a in (x for pair in arrays for x in pair):
            lo = a.ctypes.data - raw.ctypes.data
            free[lo:lo + a.nbytes] = False
        assert page.ctypes.data % PAGE == 0 and free.sum() == raw.size - (21 * nn + N * nn + 88 * npf + 80 * npf)
        meets = [Meet(2) for _ in range(3)]

        def lane(i):
            par, out = arrays[i]

            def evaluate(ctx, ev):
                out.view(np.uint8)[:] = FILL
                if i == 0:
                    ctx.call(ev.evaluate_gpu, par, nn * N, out)
                    got = masked(out.reshape(nn, N), po.nq_live_mask(nqv, N), nn)
                else:
                    ctx.call(ev.evaluate_gpu, par, npf * 20, OPT14, "lb1", out)
                    got = masked(out.reshape(npf, 20), po.pfsp_live_mask(pfv, 20), npf)
                clean = not raw[free].any() and par.tobytes() == (nq_par if i == 0 else pf_par).tobytes()
                ctx.record("eval", ctx.call(lambda: ev.last_xfer), clean, got)

            def job(ctx):
                ev = ctx.call(tsb200.NQueensEvaluator, N, 1, nn) if i == 0 else \
                    ctx.call(lambda: tsb200.PfspEvaluator(14, tables=t, M=npf))
                try:
                    yield meets[0]
                    ctx.call(ev.register_host, par)
                    ctx.call(ev.register_host, out)
                    for _ in range(REG_LOOPS):
                        evaluate(ctx, ev)
                    yield meets[1]
                    if i == first:
                        ctx.call(ev.unregister_host, par)
                        ctx.call(ev.unregister_host, out)
                    for _ in range(REG_LOOPS):
                        evaluate(ctx, ev)
                    yield meets[2]
                    if i != first:
                        ctx.call(ev.unregister_host, par)
                        ctx.call(ev.unregister_host, out)
                    evaluate(ctx, ev)
                finally:
                    ctx.call(ev.close)
            return job
        return [lane(0), lane(1)]

    want = []
    for i, w in enumerate((want_nq, want_pf)):
        second = R_IN | R_OUT if i == first else R_ZC
        want.append([("eval", R_ZC, True, w)] * REG_LOOPS + [("eval", second, True, w)] * REG_LOOPS
                    + [("eval", R_IN | R_OUT, True, w)])
    check_scenario(f"7 two handles, one page, lane {first} unregisters first", jobs, want)

"""GPU tests of the PFSP bound kernels on every machine count and every value-range route (`pytest -m gpu`).

tsb_pfsp_create picks kernel specialisations from the tables it is given: the template machine count (5, 10 or 20,
fewer machines zero-padded), lb1 / lb1_d with two children per register (16-bit lanes) or one, lb2 on the
one-word-per-use table or the packed one, or no lb2 at all.  The instances of tests/golden/pfsp_shapes.npz
(make_golden_shapes.py) each aim at one of these routes; every test asserts the route (PfspEvaluator.route) it means
to exercise and compares the bounds BIT-EXACTLY with the reference's own values from the fixture and with the oracle
on seeded random chunks.  Only live slots (k >= limit1 + 1) are compared."""
import zlib

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po
from oracle import pyoracle50 as po50
from test_gpu_parity import copy_tables
from test_oracle import SHAPE_TAGS, SHAPES, shape_evaluate, shape_parents, shape_tables

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
INT64_MAX = 2**63 - 1
ROUTE_BITS = tsb200.ROUTE_SIMD16 | tsb200.ROUTE_LB2 | tsb200.ROUTE_LB2U
# instances with <= 10 machines on the 20-job handle: the ones whose route the environment switches can change
SMALL_TAGS = [t for t in SHAPE_TAGS if t.startswith("j20_") and int(t[-2:]) <= 10]
# one instance per route for the fused expand and the device pool (1, 3, 4, 7 and 13 machines across the value
# classes): the scalar lb1 count kernels and the packed-table lb2 count kernel on 5, 10 and 20 template machines
# (j20_rs_m04, j20_rs_m07, j20_rs_m13), the one-word-table lb2 count kernel on 5 and 10 (j20_pk_m03, j20_pk_m07)
EXPAND_TAGS = ["j20_tl_m01", "j20_se65536_m01", "j20_pk_m03", "j20_wd_m03", "j20_rs_m04", "j20_pk_m07", "j20_rs_m07",
               "j20_tl_m13", "j20_rs_m13", "j20_wd_m13", "j20_te2047_m18"]
# the settings of TSB200_NO_SIMD16 / TSB200_NO_LB2U that move an instance off its default route
FORCED = [(True, False), (False, True), (True, True)]


@pytest.fixture(scope="module", autouse=True)
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


@pytest.fixture(scope="module")
def shapes():
    return np.load(SHAPES)


@pytest.fixture(autouse=True)
def default_routes(monkeypatch):
    """no environment switch of tsb_pfsp_create leaks in from the caller's environment"""
    monkeypatch.delenv("TSB200_NO_SIMD16", raising=False)
    monkeypatch.delenv("TSB200_NO_LB2U", raising=False)


def describe(route):
    return (f"mt={route & tsb200.ROUTE_MT_MASK} simd16={int(bool(route & tsb200.ROUTE_SIMD16))} "
            f"lb2={int(bool(route & tsb200.ROUTE_LB2))} lb2u={int(bool(route & tsb200.ROUTE_LB2U))}")


def open_handle(g, tag, M):
    """(evaluator, oracle tables): a handle created from the tables the oracle builds for the instance (Chapel
    min_heads, the tables of the Taillard path)"""
    t = shape_tables(g, tag, heads_mode=0)
    cls = tsb200.PfspTables50 if t.jobs > po.MAX_JOBS else tsb200.PfspTables
    return tsb200.PfspEvaluator(tables=copy_tables(t, cls), M=M), t


def rand_nodes(rng, jobs, count, depth_lo=0):
    """seeded nodes of depth depth_lo .. jobs-1 (depth 0: the root, limit1 = -1)"""
    nodes = np.zeros(count, dtype=tsb200.PFSP_NODE50_DTYPE if jobs > po.MAX_JOBS else tsb200.PFSP_NODE_DTYPE)
    depth = rng.integers(depth_lo, jobs, size=count)
    nodes["depth"], nodes["limit1"] = depth, depth - 1
    nodes["prmu"][:, :jobs] = np.argsort(rng.random((count, jobs)), axis=1).astype(np.int32)
    return nodes


def oracle_dtype(jobs):
    return po50.PFSP_NODE_DTYPE if jobs > po.MAX_JOBS else po.PFSP_NODE_DTYPE


def gpu_live(ev, parents, lb, best):
    got = ev.evaluate(parents, lb, best).reshape(-1, ev.jobs)
    return got[po.pfsp_live_mask(parents.view(oracle_dtype(ev.jobs)), ev.jobs)]


def check_oracle(ev, t, parents, lb, best, msg=""):
    want = shape_evaluate(t, tsb200.LB_NAMES[lb], parents.view(oracle_dtype(t.jobs)), best)
    np.testing.assert_array_equal(gpu_live(ev, parents, lb, best), want, err_msg=f"{lb} best={best} {msg}")


def check_fixture(ev, g, tag, lb2=True):
    """the fixture's nodes: lb1 / lb1_d, lb2 at every incumbent of the fixture (plus the int64 maximum and a value
    below INT32_MIN, which the library clamps to the int32 range), and lb1_d of the root"""
    parents = shape_parents(g, tag)
    np.testing.assert_array_equal(gpu_live(ev, parents, "lb1", INT_MAX), g[f"{tag}_lb1"], err_msg="lb1")
    np.testing.assert_array_equal(gpu_live(ev, parents, "lb1_d", INT_MAX), g[f"{tag}_lb1_d"], err_msg="lb1_d")
    if lb2 and ev.route & tsb200.ROUTE_LB2:
        bests = [int(b) for b in g[f"{tag}_lb2_bests"]]
        want = g[f"{tag}_lb2"]
        for i, best in enumerate(bests):
            np.testing.assert_array_equal(gpu_live(ev, parents, "lb2", best), want[i], err_msg=f"lb2 best={best}")
        assert bests[0] == INT_MAX and bests[-1] == -1  # (every bound is >= 0: below it the exit is at the first pair)
        np.testing.assert_array_equal(gpu_live(ev, parents, "lb2", INT64_MAX), want[0], err_msg="lb2 best=2^63-1")
        np.testing.assert_array_equal(gpu_live(ev, parents, "lb2", -2**40), want[-1], err_msg="lb2 best=-2^40")
    if f"{tag}_root_lb1_d" in g:
        root = np.zeros(1, dtype=tsb200.PFSP_NODE_DTYPE)
        root["limit1"] = -1
        root["prmu"][0, :] = np.arange(20)
        np.testing.assert_array_equal(gpu_live(ev, root, "lb1_d", INT_MAX), g[f"{tag}_root_lb1_d"], err_msg="root")


def median_bound(g, tag):
    """the median lb2 bound at best = INT_MAX over the live slots of the fixture's nodes (the middle incumbent
    make_golden_shapes.py derives from them)"""
    vals = np.sort(g[f"{tag}_lb2"][0])  # (row 0: best = INT_MAX)
    return int(vals[int(0.5 * (vals.size - 1))])


def assert_refuses_lb2(ev, parents):
    with pytest.raises(tsb200.TsbError) as e:
        ev.evaluate(parents, "lb2", INT_MAX)
    assert e.value.code == tsb200._lib.EINVAL


@pytest.mark.parametrize("tag", SHAPE_TAGS)
def test_fixture_instance(shapes, tag):
    """every instance on its own route: the reference's bounds from the fixture, then seeded chunks of ragged sizes
    (every depth, roots included) against the oracle"""
    g = shapes
    jobs = int(g[f"{tag}_dims"][0])
    ev, t = open_handle(g, tag, M=4000)
    with ev:
        want_route = int(g[f"{tag}_route"][0])
        assert ev.route == want_route, f"{describe(ev.route)} != {describe(want_route)}"
        check_fixture(ev, g, tag)
        rng = np.random.default_rng(zlib.crc32(tag.encode()))
        lb2 = bool(ev.route & tsb200.ROUTE_LB2)
        mid = median_bound(g, tag) if lb2 else None
        for count in (1, 63, 64, 65, 127, 128, 129, 3000):
            parents = rand_nodes(rng, jobs, count)
            check_oracle(ev, t, parents, "lb1_d", INT_MAX, f"count={count}")
            check_oracle(ev, t, parents, "lb1", INT_MAX, f"count={count}")
            if lb2 and (jobs <= po.MAX_JOBS or count < 3000):
                check_oracle(ev, t, parents, "lb2", INT_MAX, f"count={count}")
                check_oracle(ev, t, parents, "lb2", mid, f"count={count}")
        if not lb2:
            assert_refuses_lb2(ev, parents)


@pytest.mark.parametrize("no_simd16,no_lb2u", FORCED)
@pytest.mark.parametrize("tag", SMALL_TAGS)
def test_forced_routes(shapes, tag, no_simd16, no_lb2u, monkeypatch):
    """TSB200_NO_SIMD16 / TSB200_NO_LB2U (read when the handle is created) move an instance with <= 10 machines to
    the scalar lb1 kernels and to the packed lb2 table: every route gives the same bounds (the default route is
    test_fixture_instance)"""
    if no_simd16:
        monkeypatch.setenv("TSB200_NO_SIMD16", "1")
    if no_lb2u:
        monkeypatch.setenv("TSB200_NO_LB2U", "1")
    g = shapes
    want_route = int(g[f"{tag}_route"][0])
    if no_simd16:
        want_route &= ~(tsb200.ROUTE_SIMD16 | tsb200.ROUTE_LB2U)
    if no_lb2u:
        want_route &= ~tsb200.ROUTE_LB2U
    ev, t = open_handle(g, tag, M=600)
    with ev:
        assert ev.route == want_route, f"{describe(ev.route)} != {describe(want_route)}"
        check_fixture(ev, g, tag)
        rng = np.random.default_rng(zlib.crc32(tag.encode()) + 2 * no_simd16 + no_lb2u)
        parents = rand_nodes(rng, 20, 600)
        for lb in ("lb1_d", "lb1") + (("lb2",) if want_route & tsb200.ROUTE_LB2 else ()):
            check_oracle(ev, t, parents, lb, INT_MAX)
        if want_route & tsb200.ROUTE_LB2:
            check_oracle(ev, t, parents, "lb2", median_bound(g, tag))


REFUSED_TAGS = [t for t in SHAPE_TAGS if not int(np.load(SHAPES)[f"{t}_route"][0]) & tsb200.ROUTE_LB2]


@pytest.mark.parametrize("tag", REFUSED_TAGS)
def test_lb2_refusal(shapes, tag):
    """a handle without lb2 (one machine, p > 127, min_tails > 2047) refuses every lb2 call with TSB_EINVAL, leaves
    its pool as it was, and still gives the oracle's lb1 / lb1_d"""
    import torch
    g = shapes
    jobs = int(g[f"{tag}_dims"][0])
    ev, t = open_handle(g, tag, M=500)
    with ev:
        assert not ev.route & tsb200.ROUTE_LB2
        rng = np.random.default_rng(zlib.crc32(tag.encode()) + 7)
        parents = rand_nodes(rng, jobs, 500)
        assert_refuses_lb2(ev, parents)
        d_par = torch.from_numpy(parents.view(np.uint8).reshape(-1)).cuda()
        d_out = torch.empty(500 * jobs, dtype=torch.int32, device="cuda")
        with pytest.raises(tsb200.TsbError) as e:
            ev.evaluate_device("lb2", d_par.data_ptr(), 500, INT_MAX, d_out.data_ptr(), 0)
        assert e.value.code == tsb200._lib.EINVAL
        if jobs <= po.MAX_JOBS:
            with pytest.raises(tsb200.TsbError) as e:
                ev.expand(parents, "lb2", INT64_MAX)
            assert e.value.code == tsb200._lib.EINVAL
            start = parents[parents["depth"] > 0][:100].copy()
            ev.pool_push(start)
            with pytest.raises(tsb200.TsbError) as e:
                ev.pool_step("lb2", 1, 500, INT64_MAX)
            assert e.value.code == tsb200._lib.EINVAL
            assert ev.pool_size == start.shape[0]
            assert ev.pool_drain().tobytes() == start.tobytes()
        for lb in ("lb1_d", "lb1"):
            check_oracle(ev, t, parents, lb, INT_MAX)


def _check_expand(ev, t, parents, lb, best):
    got, gsol, gbest = ev.expand(parents, lb, best)
    want, wsol, wbest = po.pfsp_expand(t, tsb200.LB_NAMES[lb], parents.view(po.PFSP_NODE_DTYPE), best)
    assert (gsol, gbest, got.shape[0]) == (wsol, wbest, want.shape[0]), (lb, best)
    assert got.tobytes() == want.tobytes(), (lb, best)
    return gbest


@pytest.mark.parametrize("tag", EXPAND_TAGS)
def test_expand_and_device_pool(shapes, tag):
    """the fused evaluate + generate_children and the device-resident pool on each route: children byte-identical to
    the oracle's evaluate + sequential generate_children, with the same incumbent after the call (best = the int64
    maximum, lowered by leaves inside the chunk, and a value from the oracle's own bounds); then a pool byte-identical
    to the reference's pool loop after 40 rounds"""
    g = shapes
    ev, t = open_handle(g, tag, M=2000)
    with ev:
        assert ev.route == int(g[f"{tag}_route"][0]), describe(ev.route)
        lbs = ("lb1", "lb1_d") + (("lb2",) if ev.route & tsb200.ROUTE_LB2 else ())
        rng = np.random.default_rng(zlib.crc32(tag.encode()) + 1)
        for count, lo in ((1, 19), (129, 10), (2000, 12)):
            parents = rand_nodes(rng, 20, count, depth_lo=lo)
            inf = shape_evaluate(t, 1, parents.view(po.PFSP_NODE_DTYPE), INT_MAX)
            for lb in lbs:
                for best in (INT64_MAX, int(np.median(inf))):
                    _check_expand(ev, t, parents, lb, best)
        assert ev.slow_rounds > 0  # leaves lowered best inside a chunk: the redone rounds are checked as well
        for lb in lbs:
            m, M, best = 25, 300, INT64_MAX
            start = rand_nodes(rng, 20, 40, depth_lo=2)
            start["depth"][:] = np.minimum(start["depth"], 6)
            start["limit1"][:] = start["depth"] - 1
            host_pool = start.copy()
            ev.pool_push(start)
            for _ in range(40):
                n_par, n_child, n_sol, best2 = ev.pool_step(lb, m, M, best)
                if host_pool.shape[0] < m:
                    assert n_par == 0
                    break
                n = min(host_pool.shape[0], M)
                chunk = np.ascontiguousarray(host_pool[host_pool.shape[0] - n:])
                kids, sol, wbest = po.pfsp_expand(t, tsb200.LB_NAMES[lb], chunk.view(po.PFSP_NODE_DTYPE), best)
                host_pool = np.concatenate([host_pool[: host_pool.shape[0] - n], kids.view(tsb200.PFSP_NODE_DTYPE)])
                assert (n_par, n_child, n_sol, best2) == (n, kids.shape[0], sol, wbest), lb
                best = best2
                assert ev.pool_size == host_pool.shape[0]
            assert best < INT64_MAX  # the pool reached leaves
            assert ev.pool_drain().tobytes() == np.ascontiguousarray(host_pool).tobytes() and ev.pool_size == 0


@pytest.mark.parametrize("lb", ["lb1_d", "lb1", "lb2"])
def test_evaluate_device_large_batch(shapes, lb):
    """300 000 parents (> M_max) of a 7-machine instance on torch's current stream: a strided sample against the
    oracle, and the bounds of a permuted batch are the permuted bounds; count == 0 is a no-op and unaligned device
    pointers are refused"""
    import torch
    tag, P = "j20_pk_m07", 300_000
    ev, t = open_handle(shapes, tag, M=1000)
    rng = np.random.default_rng(7)
    parents = rand_nodes(rng, 20, P)
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    best = median_bound(shapes, tag)
    with ev:
        assert ev.route == int(shapes[f"{tag}_route"][0])
        d_par = torch.from_numpy(parents.view(np.uint8).reshape(-1)).to(dev)
        d_out = torch.empty(P * 20, dtype=torch.int32, device=dev)
        ev.evaluate_device(lb, d_par.data_ptr(), P, best, d_out.data_ptr(), stream)
        torch.cuda.synchronize()
        got = d_out.cpu().numpy().reshape(P, 20)
        idx = np.arange(0, P, 97)
        sample = np.ascontiguousarray(parents[idx])
        live = po.pfsp_live_mask(sample.view(po.PFSP_NODE_DTYPE), 20)
        want = shape_evaluate(t, tsb200.LB_NAMES[lb], sample.view(po.PFSP_NODE_DTYPE), best)
        np.testing.assert_array_equal(got[idx][live], want)
        perm = rng.permutation(P)
        d_par2 = torch.from_numpy(np.ascontiguousarray(parents[perm]).view(np.uint8).reshape(-1)).to(dev)
        d_out2 = torch.empty_like(d_out)
        ev.evaluate_device(lb, d_par2.data_ptr(), P, best, d_out2.data_ptr(), stream)
        torch.cuda.synchronize()
        live_all = po.pfsp_live_mask(parents[perm].view(po.PFSP_NODE_DTYPE), 20)
        np.testing.assert_array_equal(d_out2.cpu().numpy().reshape(P, 20)[live_all], got[perm][live_all])
        d_out2.fill_(-7)
        ev.evaluate_device(lb, d_par.data_ptr(), 0, best, d_out2.data_ptr(), stream)
        torch.cuda.synchronize()
        assert (d_out2 == -7).all()
        for par, out in ((d_par.data_ptr() + 4, d_out.data_ptr()), (d_par.data_ptr(), d_out.data_ptr() + 4)):
            with pytest.raises(tsb200.TsbError) as e:
                ev.evaluate_device(lb, par, 10, best, out, stream)
            assert e.value.code == tsb200._lib.EALIGN

"""tsb_pfsp_pool_run (PfspEvaluator.pool_run): the PFSP offload loop in launches of the persistent kernel
(csrc/pfsp_rounds.cuh) for lb1 / lb1_d, the loop of tsb_pfsp_pool_step otherwise.  Every route must give exactly the
rounds of tsb_pfsp_pool_step: the same counters, the same incumbent, the same pool after every call, byte for byte."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po
from test_gpu_parity import rand_pfsp
from tsb200 import _lib

OPT = {1: 1278, 14: 1377, 20: 1591, 21: 2297}
INT64_MAX = 2**63 - 1


def _root(jobs=20):
    """the 380 depth-2 nodes of the tree (the root's grandchildren), enough for m = 25"""
    nodes = np.zeros(jobs * (jobs - 1), dtype=tsb200.PFSP_NODE_DTYPE)
    x = 0
    for i in range(jobs):
        for j in range(1, jobs):
            prmu = np.arange(jobs)
            prmu[[0, i]] = prmu[[i, 0]]
            prmu[[1, j]] = prmu[[j, 1]]
            nodes["prmu"][x, :jobs] = prmu
            x += 1
    nodes["depth"], nodes["limit1"] = 2, 1
    return nodes


def _steps(ev, lb, m, M, best, max_rounds):
    """pool_step rounds, summed like pool_run's counters"""
    tot = [0, 0, 0, 0]
    for _ in range(max_rounds):
        n_par, n_child, n_sol, best = ev.pool_step(lb, m, M, best)
        if n_par == 0:
            break
        tot = [tot[0] + 1, tot[1] + n_par, tot[2] + n_child, tot[3] + n_sol]
    return tot, best


def _run_vs_steps(inst, lb, m, M, best, start, calls=(1, 3, 20)):
    """two handles with the same start pool: pool_run in calls of `calls` rounds against as many pool_step rounds"""
    with tsb200.PfspEvaluator(inst, M=M) as a, tsb200.PfspEvaluator(inst, M=M) as b:
        a.pool_push(start)
        b.pool_push(start)
        best_a = best_b = best
        for k in calls:
            want, best_a = _steps(a, lb, m, M, best_a, k)
            got = b.pool_run(lb, m, M, best_b, max_rounds=k)
            best_b = got[4]
            assert list(got[:4]) == want and best_b == best_a, (k, got, want, best_a)
            assert b.pool_size == a.pool_size
        assert b.pool_drain().tobytes() == a.pool_drain().tobytes()
        return {"route": b.route, "slow_rounds": b.slow_rounds, "launches": (a.kernel_launches, b.kernel_launches)}


def _start(inst, best, seed):
    if best != INT64_MAX:
        return _root()
    # from the root, no incumbent prunes nothing: deep random nodes keep the tree small, and their leaves lower best
    # in many rounds (IMPROVED exits of the persistent kernel)
    return rand_pfsp(np.random.default_rng(seed), 20, 2000, depth_lo=13)


@pytest.mark.gpu
@pytest.mark.parametrize("scalar", [False, True], ids=["simd16", "scalar"])
@pytest.mark.parametrize("best", ["opt", "max"])
@pytest.mark.parametrize("m,M", [(5, 300), (25, 6000), (25, 20000), (25, 50000)])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
@pytest.mark.parametrize("inst", [1, 14, 21])
def test_pool_run_equals_pool_steps(inst, lb, m, M, best, scalar, monkeypatch):
    if scalar:
        monkeypatch.setenv("TSB200_NO_SIMD16", "1")
    b0 = OPT[inst] if best == "opt" else INT64_MAX
    r = _run_vs_steps(inst, lb, m, M, b0, _start(inst, b0, 100 + inst))
    if scalar:
        assert not (r["route"] & tsb200.ROUTE_SIMD16)
    if best == "max":
        assert r["slow_rounds"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("best", [1377, 2**31 - 1])
@pytest.mark.parametrize("M", [300, 6000])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_pool_run_against_the_oracle_rule(lb, M, best):
    """pool_run(max_rounds=k) against po.pfsp_expand applied round by round to a host pool"""
    inst, m = 14, 25
    t = po.tables(inst, heads_mode=0)
    rng = np.random.default_rng(12)
    start = rand_pfsp(rng, 20, 40, depth_lo=2)
    start["depth"][:] = np.minimum(start["depth"], 6)
    start["limit1"][:] = start["depth"] - 1
    host_pool = start.copy()
    with tsb200.PfspEvaluator(inst, M=M) as ev:
        ev.pool_push(start)
        for k in (1, 2, 5, 13):
            got = ev.pool_run(lb, m, M, best, max_rounds=k)
            want = [0, 0, 0, 0]
            for _ in range(k):
                if host_pool.shape[0] < m:
                    break
                n = min(host_pool.shape[0], M)
                chunk = np.ascontiguousarray(host_pool[host_pool.shape[0] - n:])
                kids, sol, best = po.pfsp_expand(t, tsb200.LB_NAMES[lb], chunk.view(po.PFSP_NODE_DTYPE), best)
                host_pool = np.concatenate([host_pool[: host_pool.shape[0] - n], kids.view(tsb200.PFSP_NODE_DTYPE)])
                want = [want[0] + 1, want[1] + n, want[2] + kids.shape[0], want[3] + sol]
            assert list(got[:4]) == want and got[4] == best, (k, got, want, best)
            assert ev.pool_size == host_pool.shape[0]
        rest = ev.pool_drain()
        assert rest.tobytes() == np.ascontiguousarray(host_pool).tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("best", ["opt", "max"])
@pytest.mark.parametrize("inst,lb,m,M", [(14, "lb1", 25, 6000), (14, "lb1_d", 5, 300), (21, "lb1", 25, 20000)])
def test_pool_run_with_arena_growth(inst, lb, m, M, best, monkeypatch):
    """a small initial arena: the kernel leaves for room (SPACE), the arena grows, the loop relaunches"""
    monkeypatch.setenv("TSB200_POOL_CAP", "4000")
    b0 = OPT[inst] if best == "opt" else INT64_MAX
    _run_vs_steps(inst, lb, m, M, b0, _start(inst, b0, 300 + inst))


def _sms():
    return tsb200.lib().tsb_device_sm_count(0)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["lb2", "above_20000", "large_M", "no_rounds"])
def test_fallbacks_equal_pool_steps(case, monkeypatch):
    """lb2, M above 20 000 (the step loop is faster there), M above the kernel's capacity (384 parents per SM) and
    TSB200_NO_ROUNDS=1 run the pool_step loop"""
    lb, M = "lb1", 6000
    if case == "lb2":
        lb, M = "lb2", 300
    elif case == "above_20000":
        M = 20001
    elif case == "large_M":
        M = 384 * _sms() + 1
    else:
        monkeypatch.setenv("TSB200_NO_ROUNDS", "1")
    r = _run_vs_steps(14, lb, 25, M, OPT[14], _root(), calls=(1, 3, 30))
    assert r["launches"][0] == r["launches"][1]  # the same two kernels per round


@pytest.mark.gpu
def test_persistent_route_takes_few_launches():
    with tsb200.PfspEvaluator(14, M=6000) as a, tsb200.PfspEvaluator(14, M=6000) as b:
        a.pool_push(_root())
        b.pool_push(_root())
        want, _ = _steps(a, "lb1", 25, 6000, OPT[14], 2**40)
        got = b.pool_run("lb1", 25, 6000, OPT[14])
        assert list(got[:4]) == want and want[0] > 20
        assert b.kernel_launches <= 2 and a.kernel_launches >= 2 * want[0]


@pytest.mark.gpu
def test_wide_handle_and_bad_arguments():
    with tsb200.PfspEvaluator(41, M=300) as ev:
        with pytest.raises(tsb200.TsbError) as e:
            ev.pool_run("lb1", 25, 300, 2991)
        assert e.value.code == _lib.EUNSUPPORTED
    with tsb200.PfspEvaluator(14, M=300) as ev:
        ev.pool_push(_root())
        for args in (("lb1", 0, 300, 1377, 5), ("lb1", 25, 0, 1377, 5), ("lb1", 25, 301, 1377, 5),
                     ("lb1", 25, 300, 1377, -1), (3, 25, 300, 1377, 5)):
            with pytest.raises(tsb200.TsbError) as e:
                ev.pool_run(*args[:4], max_rounds=args[4])
            assert e.value.code == _lib.EINVAL
        assert ev.pool_size == 380


def test_null_handle_is_einval():
    u = C.c_uint64(0)
    b = C.c_int64(1377)
    L = tsb200.lib()
    assert L.tsb_pfsp_pool_run(None, 1, 25, 300, 5, C.byref(b), C.byref(u), C.byref(u), C.byref(u), C.byref(u)) == _lib.EINVAL


@pytest.mark.gpu
def test_ta014_lb1_search_at_M_20000_runs_in_the_persistent_kernel(golden_dir, monkeypatch):
    monkeypatch.setenv("TSB200_NO_STEAL", "1")
    st = tsb200.pfsp_search_device(14, "lb1", 1, 25, 20000, 1)
    ref = po.pfsp_search_offload(14, tsb200.LB_NAMES["lb1"], 1, 25, 20000, 1)
    assert (st.explored_tree, st.explored_sol, st.best) == (ref.tree, ref.sol, ref.best)
    assert (st.offloads, st.offloaded_parents) == (ref.offloads, ref.offloaded_parents)
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["pfsp"]["ta014_lb1_ub1"]
    assert (st.explored_tree, st.explored_sol, st.best) == (counts["tree"], counts["sol"], counts["best"])
    assert 4 * st.kernel_launches <= st.offloads


@pytest.mark.gpu
def test_ta020_lb1d_at_the_default_M(golden_dir):
    gold = json.load(open(os.path.join(golden_dir, "pfsp_chapel_heads.json")))["counts"].get("ta020_lb1d")
    if not gold:
        pytest.skip("golden count not generated (make_golden_chapel.py --no-ta020)")
    assert (gold["tree"], gold["sol"], gold["best"]) == (836490312, 3764, 1591)
    with tsb200.PfspEvaluator(20, M=50000) as ev:
        st = ev.search(20, "lb1_d", 1, 25, 50000)
    assert (st.explored_tree, st.explored_sol, st.best) == (gold["tree"], gold["sol"], gold["best"])


@pytest.mark.gpu
@pytest.mark.parametrize("D", [3, 8])
def test_stealing_with_the_persistent_kernel(golden_dir, D):
    st = tsb200.pfsp_search_device(14, "lb1", 1, 25, 20000, D)
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["pfsp"]["ta014_lb1_ub1"]
    assert (st.explored_tree, st.explored_sol, st.best) == (counts["tree"], counts["sol"], counts["best"])

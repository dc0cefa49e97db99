"""GPU parity tests (`pytest -m gpu`).  Every comparison goes through the C ABI
(libtsb200.so via the tsb200 binding) and is BIT-EXACT against the CPU oracle on the same seeded
inputs, against the committed golden vectors produced by the reference's own C sources, and — for whole
searches — against the counts the reference binaries print.  Only live slots (k >= depth resp.
k >= limit1+1) are compared: the slots below the live range are unspecified in the reference (its
kernels do not write them, its consumer does not read them) and in this library."""
import json
import os

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1


def _require_gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device (and must not fall back to the CPU)"


@pytest.fixture(scope="module", autouse=True)
def gpu():
    _require_gpu()


def rand_nq(rng, N, count, depth_lo=0, depth_hi=None):
    depth_hi = N if depth_hi is None else depth_hi
    nodes = np.zeros(count, dtype=tsb200.NQ_NODE_DTYPE)
    nodes["depth"] = rng.integers(depth_lo, depth_hi + 1, size=count)
    # row-wise random permutations of 0..N-1
    keys = rng.random((count, N))
    nodes["board"][:, :N] = np.argsort(keys, axis=1).astype(np.uint8)
    return nodes


def rand_pfsp(rng, jobs, count, depth_lo=1):
    nodes = np.zeros(count, dtype=tsb200.PFSP_NODE_DTYPE)
    depth = rng.integers(depth_lo, jobs, size=count)  # depth_lo .. jobs-1
    nodes["depth"] = depth
    nodes["limit1"] = depth - 1
    nodes["prmu"][:, :jobs] = np.argsort(rng.random((count, jobs)), axis=1).astype(np.int32)
    return nodes


def check_nq(ev, parents, N):
    got = ev.evaluate(parents).reshape(-1, N)
    want = po.nq_evaluate(parents.view(po.NQ_NODE_DTYPE), N).reshape(-1, N)
    live = po.nq_live_mask(parents.view(po.NQ_NODE_DTYPE), N)
    np.testing.assert_array_equal(got[live], want[live])
    return got


def copy_tables(src, cls):
    """the same PFSP tables in another ctypes mirror of the layout: oracle Tables <-> tsb200.PfspTables (20 jobs),
    pyoracle50.Tables <-> tsb200.PfspTables50"""
    t = cls()
    for name in ("jobs", "machines", "pairs"):
        setattr(t, name, getattr(src, name))
    for name in ("p_times", "min_heads", "min_tails", "johnson", "lags", "mp0", "mp1", "mp_order"):
        np.ctypeslib.as_array(getattr(t, name))[:] = np.ctypeslib.as_array(getattr(src, name))
    return t


def check_pfsp(ev, parents, lb, best):
    jobs = ev.jobs
    got = ev.evaluate(parents, lb, best).reshape(-1, jobs)
    t = copy_tables(ev.tables, po.Tables)  # the oracle gets the very same tables the device got (an input of the kernels)
    kind = tsb200.LB_NAMES[lb]
    want = po.pfsp_evaluate(t, kind, parents.view(po.PFSP_NODE_DTYPE), best).reshape(-1, jobs)
    live = po.pfsp_live_mask(parents.view(po.PFSP_NODE_DTYPE), jobs)
    np.testing.assert_array_equal(got[live], want[live])
    return got


# ------------------------------------------------------------------------------------------ N-Queens
@pytest.mark.parametrize("N", [1, 4, 8, 13, 14, 16, 17, 19, 20])
def test_nq_random_all_depths(N):
    rng = np.random.default_rng(1000 + N)
    with tsb200.NQueensEvaluator(N, M=70000) as ev:
        for count in (1, 3, 511, 512, 513, 4096 + 17, 50000, 65537):
            check_nq(ev, rand_nq(rng, N, count), N)
        assert ev.kernel_launches == 8


@pytest.mark.parametrize("N", [5, 8, 14, 17, 19, 20])
def test_nq_golden_vectors_from_reference(golden_dir, N):
    gold = np.load(os.path.join(golden_dir, "nqueens_labels.npz"))
    parents = gold[f"parents_N{N}"].view(tsb200.NQ_NODE_DTYPE)
    want = gold[f"labels_N{N}"].reshape(-1, N)
    with tsb200.NQueensEvaluator(N, g=3, M=parents.shape[0]) as ev:  # g never changes results
        got = ev.evaluate(parents).reshape(-1, N)
    live = po.nq_live_mask(parents.view(po.NQ_NODE_DTYPE), N)
    np.testing.assert_array_equal(got[live], want[live])


def test_nq_edge_cases():
    N = 17
    with tsb200.NQueensEvaluator(N, M=1000) as ev:
        # count == 0 is a no-op
        ev.evaluate_gpu(np.zeros(0, dtype=tsb200.NQ_NODE_DTYPE), 0, np.zeros(0, dtype=np.uint8))
        # depth == N writes no live slot; depth == 0 (root) makes every slot safe
        nodes = rand_nq(np.random.default_rng(5), N, 64)
        nodes["depth"][:32] = N
        nodes["depth"][32:] = 0
        got = check_nq(ev, nodes, N)
        assert got[32:].all()
        # count > M_max is refused, not truncated
        with pytest.raises(tsb200.TsbError):
            ev.evaluate(rand_nq(np.random.default_rng(6), N, 1001))
        # unaligned host pointers are fine on the host path
        buf = np.zeros(21 * 100 + 1, dtype=np.uint8)
        view = buf[1:].view(tsb200.NQ_NODE_DTYPE)
        view[:] = rand_nq(np.random.default_rng(7), N, 100)
        check_nq(ev, view, N)


@pytest.mark.parametrize("mode", [tsb200.XFER_AUTO, tsb200.XFER_MEMCPY, tsb200.XFER_ZEROCOPY])
@pytest.mark.parametrize("registered", [False, True])
def test_nq_transfer_modes(mode, registered):
    """driver-style use: `parents` / `labels` allocated once, optionally page-locked with register_host (then
    AUTO / ZEROCOPY run the kernel directly on them over PCIe); unregistered arrays take the staging path"""
    N, M = 17, 300000  # > the two-stream pipelining threshold of the copy path
    rng = np.random.default_rng(77)
    with tsb200.NQueensEvaluator(N, M=M) as ev:
        ev.set_xfer(mode)
        parents = np.zeros(M, dtype=tsb200.NQ_NODE_DTYPE)
        labels = np.empty(M * N, dtype=np.uint8)
        if registered:
            ev.register_host(parents)
            ev.register_host(labels)
            ev.register_host(labels)  # registering a registered range again is a no-op
        for count in (50000, 1234, M, 7):
            parents[:count] = rand_nq(rng, N, count)
            labels[:] = 7
            ev.evaluate_gpu(parents, count * N, labels)
            want = po.nq_evaluate(parents[:count].view(po.NQ_NODE_DTYPE), N).reshape(-1, N)
            live = po.nq_live_mask(parents[:count].view(po.NQ_NODE_DTYPE), N)
            np.testing.assert_array_equal(labels[: count * N].reshape(-1, N)[live], want[live])
        if registered:
            ev.unregister_host(parents)
            ev.unregister_host(labels)
            with pytest.raises(tsb200.TsbError):
                ev.unregister_host(labels)  # not registered any more


def test_nq_fresh_arrays_every_call_never_stale():
    """regression (ADVICE r1): nothing stays page-locked behind the caller's back, so arrays that are freed and
    re-allocated at the same addresses between calls are always read / written through the current mapping"""
    N = 17
    rng = np.random.default_rng(78)
    with tsb200.NQueensEvaluator(N, M=400000) as ev:
        for it in range(6):
            count = 400000 if it % 2 == 0 else 300000
            parents = rand_nq(rng, N, count)       # fresh (large: mmap'ed) arrays each iteration, freed after
            check_nq(ev, parents, N)               # ev.evaluate allocates a fresh labels array as well
            del parents
        # explicit registration with caller-owned lifetime: unregister before the array goes away
        parents = rand_nq(rng, N, 400000)
        ev.register_host(parents)
        check_nq(ev, parents, N)
        ev.unregister_host(parents)
        del parents
        check_nq(ev, rand_nq(rng, N, 400000), N)


def test_nq_without_host_registration(monkeypatch):
    monkeypatch.setenv("TSB200_NO_REGISTER", "1")  # register_host becomes a no-op
    N = 14
    with tsb200.NQueensEvaluator(N, M=20000) as ev:
        parents = rand_nq(np.random.default_rng(3), N, 20000)
        ev.register_host(parents)
        check_nq(ev, parents, N)
        ev.unregister_host(parents)


@pytest.mark.parametrize("N,which", [(12, 3), (14, 100), (15, 40)])
def test_nq_captured_real_chunks(N, which):
    """chunks exactly as the reference driver's popBackBulk hands them to evaluate_gpu"""
    parents = po.nq_capture_chunk(N, which).view(tsb200.NQ_NODE_DTYPE)
    assert parents.shape[0] > 1000
    with tsb200.NQueensEvaluator(N, M=50000) as ev:
        check_nq(ev, parents, N)


def test_nq_device_resident_large_batch():
    """4 194 304 parents (SURVEY §8d): checked against the oracle on a strided sample and by an
    order-independent property: labels of a permuted batch are the permutation of the labels"""
    import torch
    N, P = 17, 1 << 22
    rng = np.random.default_rng(17)
    parents = rand_nq(rng, N, P, depth_lo=8)
    dev = torch.device("cuda:0")
    d_par = torch.from_numpy(parents.view(np.uint8).reshape(-1)).to(dev)
    d_lab = torch.empty(P * N, dtype=torch.uint8, device=dev)
    with tsb200.NQueensEvaluator(N, M=1) as ev:
        ev.evaluate_device(d_par.data_ptr(), P, d_lab.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        got = d_lab.cpu().numpy().reshape(P, N)
        idx = np.arange(0, P, 97)
        want = po.nq_evaluate(np.ascontiguousarray(parents[idx]).view(po.NQ_NODE_DTYPE), N).reshape(-1, N)
        live = po.nq_live_mask(parents[idx].view(po.NQ_NODE_DTYPE), N)
        np.testing.assert_array_equal(got[idx][live], want[live])
        perm = rng.permutation(P)
        d_par2 = torch.from_numpy(np.ascontiguousarray(parents[perm]).view(np.uint8).reshape(-1)).to(dev)
        d_lab2 = torch.empty_like(d_lab)
        ev.evaluate_device(d_par2.data_ptr(), P, d_lab2.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        live_all = po.nq_live_mask(parents[perm].view(po.NQ_NODE_DTYPE), N)
        np.testing.assert_array_equal(d_lab2.cpu().numpy().reshape(P, N)[live_all], got[perm][live_all])
        # unaligned device pointers are refused
        with pytest.raises(tsb200.TsbError):
            ev.evaluate_device(d_par.data_ptr() + 1, 10, d_lab.data_ptr(), 0)


@pytest.mark.parametrize("N,m,M,D", [(10, 25, 50000, 1), (12, 25, 50000, 1), (12, 5, 300, 1), (13, 25, 50000, 2),
                                     (13, 7, 1000, 4), (14, 25, 50000, 1)])
def test_nq_full_search_counts(golden_dir, N, m, M, D):
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"][str(N)]
    st = tsb200.nqueens_search(N, 1, m, M, D)
    assert (st.explored_tree, st.explored_sol) == (counts["tree"], counts["sol"])
    assert st.kernel_launches == st.offloads > 0
    assert sum(st.per_gpu_tree[:D]) <= st.explored_tree


# ------------------------------------------------------------------------------------------ PFSP
@pytest.mark.parametrize("inst", [1, 14, 20, 21])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d", "lb2"])
def test_pfsp_random_nodes(inst, lb):
    rng = np.random.default_rng(inst * 10 + len(lb))
    best = int(tsb200.lib().tsb_taillard_best_ub(inst))
    with tsb200.PfspEvaluator(inst, M=20000) as ev:
        sizes = (1, 127, 128, 129, 5000, 20000) if lb != "lb2" else (1, 129, 3000)
        for count in sizes:
            parents = rand_pfsp(rng, ev.jobs, count)
            check_pfsp(ev, parents, lb, best)
            if lb == "lb2":
                check_pfsp(ev, parents, lb, INT_MAX)      # early exit disabled
                check_pfsp(ev, parents, lb, 2**63 - 1)    # Chapel's max(int) under --ub 0
                check_pfsp(ev, parents, lb, best - 200)   # aggressive early exit


@pytest.mark.parametrize("inst", [14, 21])
@pytest.mark.parametrize("lb", ["lb1", "lb1_d"])
def test_pfsp_scalar_children_formulation(inst, lb, monkeypatch):
    """TSB200_NO_SIMD16 selects the one-child-per-register formulation (the route for tables whose values do not
    fit 16 bits or whose min_tails is not non-increasing); both routes must give the oracle's bounds"""
    monkeypatch.setenv("TSB200_NO_SIMD16", "1")
    rng = np.random.default_rng(inst)
    with tsb200.PfspEvaluator(inst, M=6000) as ev:
        parents = rand_pfsp(rng, ev.jobs, 6000)
        parents["depth"][:50] = 0
        parents["limit1"][:50] = -1
        check_pfsp(ev, parents, lb, 10**9)


def test_pfsp_custom_tables_with_rising_tails():
    """min_tails that is NOT non-increasing (not what fill_min_heads_tails produces, but the C ABI takes arbitrary
    arrays): lb1 and lb1_d then differ in value, and each must match its own oracle function"""
    t = tsb200.taillard_tables(14)
    for k in range(t.machines):
        t.min_tails[k] = 40 + 37 * ((k * 7) % 5)
    rng = np.random.default_rng(3)
    with tsb200.PfspEvaluator(tables=t, M=4000) as ev:
        parents = rand_pfsp(rng, 20, 4000)
        a = check_pfsp(ev, parents, "lb1", 10**9)
        b = check_pfsp(ev, parents, "lb1_d", 10**9)
        live = po.pfsp_live_mask(parents.view(po.PFSP_NODE_DTYPE), 20)
        assert (a[live] != b[live]).any()


@pytest.mark.parametrize("inst", [1, 14, 20, 21])
def test_pfsp_golden_vectors_from_reference(golden_dir, inst):
    gold = np.load(os.path.join(golden_dir, "pfsp_bounds.npz"))
    tag = f"ta{inst:03d}"
    parents = gold[f"{tag}_parents"].view(tsb200.PFSP_NODE_DTYPE)
    best = int(tsb200.lib().tsb_taillard_best_ub(inst))
    with tsb200.PfspEvaluator(inst, M=parents.shape[0]) as ev:
        jobs = ev.jobs
        live = po.pfsp_live_mask(parents.view(po.PFSP_NODE_DTYPE), jobs)
        for lb, key, b in (("lb1", "lb1", best), ("lb1_d", "lb1_d", best), ("lb2", "lb2_best", best),
                           ("lb2", "lb2_inf", INT_MAX)):
            got = ev.evaluate(parents, lb, b).reshape(-1, jobs)
            np.testing.assert_array_equal(got[live], gold[f"{tag}_{key}"].reshape(-1, jobs)[live], err_msg=key)


def test_pfsp_root_uses_min_heads(golden_dir):
    """limit1 == -1 is only ever evaluated by lb1_d (SURVEY A.1): front = min_heads as handed to create; the values
    are those of the reference's C code built with the Chapel statement (tests/golden/pfsp_chapel_heads.json)"""
    gold = json.load(open(os.path.join(golden_dir, "pfsp_chapel_heads.json")))
    for inst in (1, 14, 20):
        with tsb200.PfspEvaluator(inst, M=16) as ev:
            root = np.zeros(1, dtype=tsb200.PFSP_NODE_DTYPE)
            root["limit1"] = -1
            root["prmu"][0, :] = np.arange(20)
            got = check_pfsp(ev, root, "lb1_d", int(tsb200.lib().tsb_taillard_best_ub(inst)))
            assert list(got.reshape(-1)[:20]) == gold["root_lb1_children_bounds"][f"ta{inst:03d}"]
            check_pfsp(ev, root, "lb1", INT_MAX)   # lb1 / lb2 on the root: children have limit1 = 0
            check_pfsp(ev, root, "lb2", INT_MAX)


@pytest.mark.parametrize("lb,which", [("lb1", 30), ("lb1_d", 30), ("lb2", 10)])
def test_pfsp_captured_real_chunks(lb, which):
    parents, best = po.pfsp_capture_chunk(14, tsb200.LB_NAMES[lb], which)
    parents = np.ascontiguousarray(parents.view(tsb200.PFSP_NODE_DTYPE))
    with tsb200.PfspEvaluator(14, M=50000) as ev:
        for registered in (False, True):
            if registered:
                ev.register_host(parents)
            for mode in (tsb200.XFER_MEMCPY, tsb200.XFER_ZEROCOPY):
                ev.set_xfer(mode)
                check_pfsp(ev, parents, lb, best)
        ev.unregister_host(parents)


@pytest.mark.parametrize("lb,D", [("lb1", 1), ("lb1_d", 1), ("lb2", 1), ("lb1", 4), ("lb2", 2)])
def test_pfsp_full_search_counts_ta014(golden_dir, lb, D):
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["pfsp"][f"ta014_lb{tsb200.LB_NAMES[lb]}_ub1"]
    st = tsb200.pfsp_search(14, lb, 1, 25, 50000, D)
    assert (st.explored_tree, st.explored_sol, st.best) == (counts["tree"], counts["sol"], counts["best"])


def test_pfsp_full_search_ta020_lb2(golden_dir):
    counts = json.load(open(os.path.join(golden_dir, "counts.json")))["pfsp"]["ta020_lb2_ub1"]
    st = tsb200.pfsp_search(20, "lb2", 1, 25, 50000, 1)
    assert (st.explored_tree, st.explored_sol, st.best) == (counts["tree"], counts["sol"], counts["best"])


@pytest.mark.parametrize("variant", ["nabeshima", "lageweg"])
@pytest.mark.parametrize("inst", [14, 21])
def test_pfsp_lb2_variants(golden_dir, variant, inst):
    """SURVEY §8(f4): LB2_NABESHIMA / LB2_LAGEWEG are pair tables handed to tsb_pfsp_create; bounds against the
    reference's C code compiled with that variant (tests/golden/pfsp_f4.npz) and against the oracle"""
    gold = np.load(os.path.join(golden_dir, "pfsp_f4.npz"))
    tag = f"{variant}_ta{inst:03d}"
    parents = gold[f"{tag}_parents"].view(tsb200.PFSP_NODE_DTYPE)
    best = int(tsb200.lib().tsb_taillard_best_ub(inst))
    with tsb200.PfspEvaluator(tables=tsb200.taillard_tables(inst, variant), M=4096) as ev:
        assert ev.tables.pairs == ev.machines - 1
        live = po.pfsp_live_mask(parents.view(po.PFSP_NODE_DTYPE), ev.jobs)
        for b, key in ((best, "lb2_best"), (INT_MAX, "lb2_inf")):
            got = ev.evaluate(parents, "lb2", b).reshape(-1, ev.jobs)
            np.testing.assert_array_equal(got[live], gold[f"{tag}_{key}"].reshape(-1, ev.jobs)[live], err_msg=key)
        rng = np.random.default_rng(inst)
        check_pfsp(ev, rand_pfsp(rng, ev.jobs, 4096), "lb2", best)
        check_pfsp(ev, rand_pfsp(rng, ev.jobs, 1000), "lb1", best)


@pytest.mark.parametrize("inst", [31, 41, 51])
def test_pfsp_max_jobs_50(golden_dir, inst):
    """SURVEY §8(f4): a MAX_JOBS = 50 handle (208-byte nodes): lb1 / lb1_d / lb2 on ta031 / ta041 / ta051 against the
    reference's C code compiled with MAX_JOBS 50 (tests/golden/pfsp_f4.npz) and against the oracle built that way"""
    from oracle import pyoracle50 as po50
    gold = np.load(os.path.join(golden_dir, "pfsp_f4.npz"))
    tag = f"jobs50_ta{inst:03d}"
    parents = gold[f"{tag}_parents"].view(tsb200.PFSP_NODE50_DTYPE)
    best = int(tsb200.lib().tsb_taillard_best_ub(inst))
    t = po50.tables(inst)
    with tsb200.PfspEvaluator(inst, M=5000) as ev:
        assert ev.wide and ev.jobs == 50
        live = po50.pfsp_live_mask(parents.view(po50.PFSP_NODE_DTYPE), 50)
        for lb, key, b in (("lb1", "lb1", best), ("lb1_d", "lb1_d", best), ("lb2", "lb2_best", best), ("lb2", "lb2_inf", INT_MAX)):
            got = ev.evaluate(parents, lb, b).reshape(-1, 50)
            np.testing.assert_array_equal(got[live], gold[f"{tag}_{key}"].reshape(-1, 50)[live], err_msg=key)
        # seeded random chunks (ragged sizes, every depth, the root for lb1_d) against the oracle
        rng = np.random.default_rng(inst)
        for count in (1, 63, 64, 65, 3000):
            nodes = np.zeros(count, dtype=tsb200.PFSP_NODE50_DTYPE)
            depth = rng.integers(0, 50, size=count)
            nodes["depth"], nodes["limit1"] = depth, depth - 1
            nodes["prmu"] = np.argsort(rng.random((count, 50)), axis=1).astype(np.int32)
            live = po50.pfsp_live_mask(nodes.view(po50.PFSP_NODE_DTYPE), 50)
            for lb, b in (("lb1_d", best), ("lb1", best)) + ((("lb2", best), ("lb2", 2**63 - 1)) if count <= 65 or inst != 51 else ()):
                if lb != "lb1_d":
                    use = nodes[nodes["limit1"] >= 0]  # lb1 / lb2 never see the root (SURVEY A.1)
                else:
                    use = nodes
                if use.shape[0] == 0:
                    continue
                got = ev.evaluate(np.ascontiguousarray(use), lb, b).reshape(-1, 50)
                want = po50.pfsp_evaluate(t, tsb200.LB_NAMES[lb], np.ascontiguousarray(use).view(po50.PFSP_NODE_DTYPE), min(b, 2**62)).reshape(-1, 50)
                lv = po50.pfsp_live_mask(use.view(po50.PFSP_NODE_DTYPE), 50)
                np.testing.assert_array_equal(got[lv], want[lv], err_msg=f"{lb} count={count}")
        # the fused expand / pool entry points are 20-job only
        with pytest.raises(tsb200.TsbError):
            ev.pool_push(np.zeros(1, dtype=tsb200.PFSP_NODE_DTYPE))

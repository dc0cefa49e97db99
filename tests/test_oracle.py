"""The CPU oracle (oracle/tsb_oracle.c) against the committed golden vectors produced by the
reference's own C sources (tests/golden/make_golden.py) and the counts its binaries print."""
import json
import os

import numpy as np
import pytest

from oracle import pyoracle as po

INT_MAX = 2**31 - 1


@pytest.fixture(scope="module")
def counts(golden_dir):
    return json.load(open(os.path.join(golden_dir, "counts.json")))


@pytest.fixture(scope="module")
def nq_gold(golden_dir):
    return np.load(os.path.join(golden_dir, "nqueens_labels.npz"))


@pytest.fixture(scope="module")
def pf_gold(golden_dir):
    return np.load(os.path.join(golden_dir, "pfsp_bounds.npz"))


@pytest.mark.parametrize("N", [5, 8, 14, 17, 19, 20])
def test_nq_labels_match_reference_isSafe(nq_gold, N):
    parents = nq_gold[f"parents_N{N}"].view(po.NQ_NODE_DTYPE)
    want = nq_gold[f"labels_N{N}"]
    for g in (1, 3):
        got = po.nq_evaluate(parents, N, g)
        np.testing.assert_array_equal(got, want)  # includes the untouched (0xCD) slots k < depth


@pytest.mark.parametrize("inst", [1, 14, 20, 21])
def test_tables_match_reference(pf_gold, inst):
    tag = f"ta{inst:03d}"
    jobs, machines, pairs = pf_gold[f"{tag}_dims"]
    t = po.tables(inst, heads_mode=1)
    assert (t.jobs, t.machines, t.pairs) == (jobs, machines, pairs)
    np.testing.assert_array_equal(t.arr("p_times", jobs * machines), pf_gold[f"{tag}_p_times"])
    np.testing.assert_array_equal(t.arr("min_heads", machines), pf_gold[f"{tag}_min_heads_C"])
    np.testing.assert_array_equal(t.arr("min_tails", machines), pf_gold[f"{tag}_min_tails"])
    np.testing.assert_array_equal(t.arr("lags", pairs * jobs), pf_gold[f"{tag}_lags"])
    np.testing.assert_array_equal(t.arr("mp0", pairs), pf_gold[f"{tag}_mp0"])
    np.testing.assert_array_equal(t.arr("mp1", pairs), pf_gold[f"{tag}_mp1"])
    # Johnson order: a permutation per pair, sorted by the same key as the reference's (ties may permute)
    ours = t.arr("johnson", pairs * jobs).reshape(pairs, jobs)
    ref = pf_gold[f"{tag}_johnson_qsort"].reshape(pairs, jobs)
    p = pf_gold[f"{tag}_p_times"].reshape(machines, jobs)
    lags = pf_gold[f"{tag}_lags"].reshape(pairs, jobs)
    for k in range(pairs):
        assert sorted(ours[k]) == list(range(jobs))
        a = p[pf_gold[f"{tag}_mp0"][k]] + lags[k]
        b = p[pf_gold[f"{tag}_mp1"][k]] + lags[k]
        key = lambda j: (0, a[j]) if a[j] < b[j] else (1, -b[j])  # noqa: E731
        assert [key(j) for j in ours[k]] == [key(j) for j in ref[k]]


def test_chapel_min_heads_known_answers(counts):
    for inst, name in ((14, "ta014"), (20, "ta020")):
        t = po.tables(inst, heads_mode=0)
        assert list(t.arr("min_heads", t.machines)) == counts["chapel_min_heads"][name]


def test_chapel_min_heads_on_reference_run_output(golden_dir):
    """the one place where the Chapel program differs from the C baseline, pinned on the output of the reference's
    own C code built with that one line rewritten to the Chapel statement (tests/golden/make_golden_chapel.py):
    min_heads of ta001..ta030 and the bounds of the root's children (the only node that reads min_heads)"""
    gold = json.load(open(os.path.join(golden_dir, "pfsp_chapel_heads.json")))
    for inst in range(1, 31):
        tag = f"ta{inst:03d}"
        t = po.tables(inst, heads_mode=0)
        assert list(t.arr("min_heads", t.machines)) == gold["min_heads"][tag]
        root = np.zeros(1, dtype=po.PFSP_NODE_DTYPE)
        root["limit1"] = -1
        root["prmu"][0, : t.jobs] = np.arange(t.jobs)
        got = po.pfsp_evaluate(t, 0, root, INT_MAX).reshape(-1)[: t.jobs]  # lb1_d: bounds[k] = lb_begin[prmu[k]]
        assert list(got) == gold["root_lb1_children_bounds"][tag]
        if inst in (14, 20):  # ... and they do differ from the C baseline's there
            c = po.tables(inst, heads_mode=1)
            assert list(c.arr("min_heads", c.machines)) != gold["min_heads"][tag]
    r = po.pfsp_search_seq(14, 0, 1, 0)
    assert (r.tree, r.sol, r.best) == tuple(gold["counts"]["ta014_lb1d"][k] for k in ("tree", "sol", "best"))


@pytest.mark.parametrize("inst", [1, 14, 20, 21])
def test_bounds_match_reference(pf_gold, inst):
    tag = f"ta{inst:03d}"
    jobs = int(pf_gold[f"{tag}_dims"][0])
    parents = pf_gold[f"{tag}_parents"].view(po.PFSP_NODE_DTYPE)
    best = int(po.lib().or_taillard_best_ub(inst))
    for heads_mode in (0, 1):  # min_heads is never read when limit1 >= 0
        t = po.tables(inst, heads_mode)
        np.testing.assert_array_equal(po.pfsp_evaluate(t, 1, parents, best), pf_gold[f"{tag}_lb1"])
        np.testing.assert_array_equal(po.pfsp_evaluate(t, 0, parents, best), pf_gold[f"{tag}_lb1_d"])
        np.testing.assert_array_equal(po.pfsp_evaluate(t, 2, parents, best), pf_gold[f"{tag}_lb2_best"])
        np.testing.assert_array_equal(po.pfsp_evaluate(t, 2, parents, INT_MAX), pf_gold[f"{tag}_lb2_inf"])
        np.testing.assert_array_equal(po.pfsp_evaluate(t, 2, parents, 2**63 - 1), pf_gold[f"{tag}_lb2_inf"])
    # root (limit1 = -1), lb1_d, C min_heads semantics
    root = np.zeros(1, dtype=po.PFSP_NODE_DTYPE)
    root["limit1"][0] = -1
    root["prmu"][0, :jobs] = np.arange(jobs)
    np.testing.assert_array_equal(po.pfsp_evaluate(po.tables(inst, 1), 0, root, best), pf_gold[f"{tag}_root_lb1_d_C"])
    # known answers: eval_solution / lb1 / lb2 on the identity permutation
    ident = np.arange(jobs, dtype=np.int32)
    t = po.tables(inst, 0)
    import ctypes as C
    p = ident.ctypes.data_as(C.c_void_p)
    kat = [po.lib().or_eval_solution(C.byref(t), p), po.lib().or_lb1_bound(C.byref(t), p, 0, jobs),
           po.lib().or_lb2_bound(C.byref(t), p, 0, jobs, INT_MAX)]
    assert kat == list(pf_gold[f"{tag}_kat"])


def test_survey_known_answers():
    t = po.tables(14, 0)
    assert list(t.arr("p_times", 20)) == [94, 43, 6, 47, 45, 51, 73, 49, 31, 58, 19, 36, 54, 75, 7, 5, 82, 20, 31, 32]
    assert list(t.arr("min_tails", 10)) == [280, 205, 115, 110, 100, 78, 50, 31, 8, 0]
    assert int(t.arr("p_times", 200).sum()) == 8930


@pytest.mark.parametrize("N", list(range(4, 13)))
def test_nq_search_counts(counts, N):
    want = counts["nqueens"][str(N)]
    assert want["sol"] == counts["nqueens_classical_solutions"][str(N)]
    r = po.nq_search_seq(N)
    assert (r.tree, r.sol) == (want["tree"], want["sol"])
    for (m, M, D) in ((25, 50000, 1), (5, 300, 1), (25, 50000, 2), (7, 1000, 4)):
        r = po.nq_search_offload(N, 1, m, M, D)
        assert (r.tree, r.sol) == (want["tree"], want["sol"]), (m, M, D)


@pytest.mark.parametrize("lb", [0, 1, 2])
def test_pfsp_search_counts_ta014(counts, lb):
    want = counts["pfsp"][f"ta014_lb{lb}_ub1"]
    for heads_mode in (0, 1):  # ta014 counts do not depend on the min_heads quirk (SURVEY A.1)
        if lb == 1 and heads_mode == 1:
            continue
        r = po.pfsp_search_seq(14, lb, 1, heads_mode)
        assert (r.tree, r.sol, r.best) == (want["tree"], want["sol"], want["best"])
    for (m, M, D) in ((25, 50000, 1), (25, 50000, 4)):
        r = po.pfsp_search_offload(14, lb, 1, m, M, D)
        assert (r.tree, r.sol, r.best) == (want["tree"], want["sol"], want["best"]), (m, M, D)


# ---- the chunk-level oracle functions the GPU expand / pool tests compare against, pinned on the driver-level ones
def _pool_search(expand, start, m, M):
    """the reference's step-2 loop (popBackBulk(m, M) -> evaluate -> generate_children -> pushBack) on a numpy pool"""
    pool, tree, sol, offloads, parents = start, 0, 0, 0, 0
    while pool.shape[0] >= m:
        n = min(pool.shape[0], M)
        chunk = np.ascontiguousarray(pool[pool.shape[0] - n:])
        kids, s = expand(chunk)
        pool = np.concatenate([pool[: pool.shape[0] - n], kids])
        tree, sol, offloads, parents = tree + kids.shape[0], sol + s, offloads + 1, parents + n
    return pool, tree, sol, offloads, parents


@pytest.mark.parametrize("N,m,M", [(10, 25, 50000), (11, 5, 300)])
def test_nq_expand_chunk_reproduces_the_offload_search(counts, N, m, M):
    """a pool driven by or_nq_expand_chunk from the warm-up pool of the driver = the driver's own step 2"""
    ref = po.nq_search_offload(N, 1, m, M, 1)
    # warm-up (step 1): breadth-first from the root until the pool holds m nodes, as the driver does
    root = np.zeros(1, dtype=po.NQ_NODE_DTYPE)
    root["board"][0, :N] = np.arange(N)
    pool, tree1, sol1 = root, 0, 0
    while pool.shape[0] < m and pool.shape[0] > 0:
        kids, s = po.nq_expand(np.ascontiguousarray(pool[:1]), N)
        pool = np.concatenate([pool[1:], kids])
        tree1, sol1 = tree1 + kids.shape[0], sol1 + s
    rest, tree2, sol2, offloads, parents = _pool_search(lambda c: po.nq_expand(c, N), pool, m, M)
    assert (offloads, parents) == (ref.offloads, ref.offloaded_parents)
    # step 3: drain what is left depth-first (order does not matter for the counts)
    tree3 = sol3 = 0
    while rest.shape[0]:
        kids, s = po.nq_expand(np.ascontiguousarray(rest), N)
        rest, tree3, sol3 = kids, tree3 + kids.shape[0], sol3 + s
    want = counts["nqueens"][str(N)]
    assert (tree1 + tree2 + tree3, sol1 + sol2 + sol3) == (want["tree"], want["sol"]) == (ref.tree, ref.sol)


@pytest.mark.parametrize("lb", [0, 1])
def test_pfsp_expand_chunk_reproduces_the_offload_search(lb):
    """or_pfsp_expand_chunk (bounds with best at launch + sequential generate_children) driven as a pool from a
    captured first chunk equals the driver emulation from that point on: same number of offloads and parents"""
    inst, m, M = 14, 25, 50000
    t = po.tables(inst, heads_mode=0)
    ref = po.pfsp_search_offload(inst, lb, 1, m, M, 1)
    first, best = po.pfsp_capture_chunk(inst, lb, 0, 1, m, M)  # the whole warm-up pool (it is < M)
    state = {"best": best}

    def expand(chunk):
        kids, s, b = po.pfsp_expand(t, lb, chunk, state["best"])
        state["best"] = b
        return kids, s

    rest, tree2, sol2, offloads, parents = _pool_search(expand, first, m, M)
    assert (offloads, parents) == (ref.offloads, ref.offloaded_parents)
    assert state["best"] == ref.best == 1377


# ------------------------------------------------------------------------------------------ SURVEY §8(f4)
def _oracle_tables_from_gold(gold, tag, Tables):
    """oracle tables whose Johnson order is the reference's own (the table is an input of the bounds)"""
    jobs, machines, pairs = (int(x) for x in gold[f"{tag}_dims"])
    t = Tables()
    t.jobs, t.machines, t.pairs = jobs, machines, pairs
    for name, key, n in (("p_times", "p_times", jobs * machines), ("min_tails", "min_tails", machines),
                         ("lags", "lags", pairs * jobs), ("johnson", "johnson_qsort", pairs * jobs),
                         ("mp0", "mp0", pairs), ("mp1", "mp1", pairs)):
        np.ctypeslib.as_array(getattr(t, name))[:n] = gold[f"{tag}_{key}"]
    np.ctypeslib.as_array(t.mp_order)[:pairs] = np.arange(pairs)
    return t


@pytest.mark.parametrize("variant", ["nabeshima", "lageweg"])
@pytest.mark.parametrize("inst", [14, 21])
def test_lb2_variants_match_reference(golden_dir, variant, inst):
    """LB2_NABESHIMA / LB2_LAGEWEG (Bound_johnson.chpl:6,36-43,50-87): the oracle's pair tables equal the ones the
    reference's fill_* produce when compiled with that variant, and its lb2 bounds equal the reference's"""
    gold = np.load(os.path.join(golden_dir, "pfsp_f4.npz"))
    tag = f"{variant}_ta{inst:03d}"
    t = po.tables(inst, 0, po.LB2_VARIANTS[variant])
    jobs, machines, pairs = (int(x) for x in gold[f"{tag}_dims"])
    assert (t.jobs, t.machines, t.pairs) == (jobs, machines, pairs) and pairs == machines - 1
    np.testing.assert_array_equal(t.arr("mp0", pairs), gold[f"{tag}_mp0"])
    np.testing.assert_array_equal(t.arr("mp1", pairs), gold[f"{tag}_mp1"])
    np.testing.assert_array_equal(t.arr("lags", pairs * jobs), gold[f"{tag}_lags"])
    parents = gold[f"{tag}_parents"].view(po.PFSP_NODE_DTYPE)
    best = int(po.lib().or_taillard_best_ub(inst))
    for tt in (t, _oracle_tables_from_gold(gold, tag, po.Tables)):  # own Johnson order and the reference's (ties)
        np.testing.assert_array_equal(po.pfsp_evaluate(tt, 2, parents, best), gold[f"{tag}_lb2_best"])
        np.testing.assert_array_equal(po.pfsp_evaluate(tt, 2, parents, INT_MAX), gold[f"{tag}_lb2_inf"])


@pytest.mark.parametrize("inst", [31, 41, 51])
def test_max_jobs_50_oracle_matches_reference(golden_dir, inst):
    """the oracle built with OR_MAX_JOBS = 50 (208-byte nodes) against the reference's C code built with MAX_JOBS 50"""
    from oracle import pyoracle50 as po50
    gold = np.load(os.path.join(golden_dir, "pfsp_f4.npz"))
    tag = f"jobs50_ta{inst:03d}"
    t = po50.tables(inst)
    jobs, machines, pairs = (int(x) for x in gold[f"{tag}_dims"])
    assert (t.jobs, t.machines, t.pairs) == (jobs, machines, pairs) and jobs == 50
    np.testing.assert_array_equal(t.arr("p_times", jobs * machines), gold[f"{tag}_p_times"])
    np.testing.assert_array_equal(t.arr("min_tails", machines), gold[f"{tag}_min_tails"])
    np.testing.assert_array_equal(t.arr("lags", pairs * jobs), gold[f"{tag}_lags"])
    parents = gold[f"{tag}_parents"].view(po50.PFSP_NODE_DTYPE)
    best = int(po.lib().or_taillard_best_ub(inst))
    np.testing.assert_array_equal(po50.pfsp_evaluate(t, 1, parents, best), gold[f"{tag}_lb1"])
    np.testing.assert_array_equal(po50.pfsp_evaluate(t, 0, parents, best), gold[f"{tag}_lb1_d"])
    np.testing.assert_array_equal(po50.pfsp_evaluate(t, 2, parents, best), gold[f"{tag}_lb2_best"])
    np.testing.assert_array_equal(po50.pfsp_evaluate(t, 2, parents, INT_MAX), gold[f"{tag}_lb2_inf"])


# ------------------------------------------------------------------------------------------ synthetic shapes
# tests/golden/pfsp_shapes.npz (tests/golden/make_golden_shapes.py): the reference's tables and bounds for synthetic
# processing-time matrices on 1..20 machines, in value classes that each select one kernel route of the device library
SHAPES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pfsp_shapes.npz")
SHAPE_TAGS = [str(x) for x in np.load(SHAPES)["tags"]]


def shape_tables(gold, tag, heads_mode=0):
    """oracle tables of fixture instance `tag` from its processing times (with its overwritten min_tails, if any)"""
    from oracle import pyoracle50 as po50
    jobs, machines, _ = (int(x) for x in gold[f"{tag}_dims"])
    mod = po50 if jobs > po.MAX_JOBS else po
    t = mod.tables_from_ptimes(gold[f"{tag}_p_times"].reshape(machines, jobs), heads_mode)
    if gold[f"{tag}_tails_set"][0]:
        np.ctypeslib.as_array(t.min_tails)[:machines] = gold[f"{tag}_min_tails"]
    return t


def shape_parents(gold, tag):
    from oracle import pyoracle50 as po50
    jobs = int(gold[f"{tag}_dims"][0])
    return gold[f"{tag}_parents"].view(po50.PFSP_NODE_DTYPE if jobs > po.MAX_JOBS else po.PFSP_NODE_DTYPE)


def shape_evaluate(t, kind, parents, best):
    """the oracle's bounds on the live slots (k >= limit1 + 1, row-major), the layout of the fixture"""
    from oracle import pyoracle50 as po50
    mod = po50 if t.jobs > po.MAX_JOBS else po
    got = mod.pfsp_evaluate(t, kind, parents, best).reshape(-1, t.jobs)
    return got[mod.pfsp_live_mask(parents, t.jobs)]


@pytest.fixture(scope="module")
def shapes():
    return np.load(SHAPES)


@pytest.mark.parametrize("tag", SHAPE_TAGS)
def test_tables_from_ptimes_match_reference(shapes, tag):
    """or_pfsp_tables_from_ptimes runs the same fill_* as the reference on any matrix (C min_heads semantics with
    heads_mode 1, the Chapel statement with heads_mode 0)"""
    g = shapes
    jobs, machines, pairs = (int(x) for x in g[f"{tag}_dims"])
    t = shape_tables(g, tag, heads_mode=1)
    assert (t.jobs, t.machines, t.pairs) == (jobs, machines, pairs)
    np.testing.assert_array_equal(t.arr("p_times", jobs * machines), g[f"{tag}_p_times"])
    np.testing.assert_array_equal(t.arr("min_heads", machines), g[f"{tag}_min_heads_C"])
    np.testing.assert_array_equal(t.arr("min_tails", machines), g[f"{tag}_min_tails"])
    np.testing.assert_array_equal(t.arr("lags", pairs * jobs), g[f"{tag}_lags"])
    np.testing.assert_array_equal(t.arr("mp0", pairs), g[f"{tag}_mp0"])
    np.testing.assert_array_equal(t.arr("mp1", pairs), g[f"{tag}_mp1"])
    if f"{tag}_min_heads_chapel" in g:
        np.testing.assert_array_equal(shape_tables(g, tag, 0).arr("min_heads", machines), g[f"{tag}_min_heads_chapel"])
    # Johnson order: a permutation per pair, sorted by the reference's key (ties may permute)
    ours = t.arr("johnson", pairs * jobs).reshape(pairs, jobs)
    ref = g[f"{tag}_johnson_qsort"].reshape(pairs, jobs)
    p = g[f"{tag}_p_times"].reshape(machines, jobs).astype(np.int64)
    lags = g[f"{tag}_lags"].reshape(pairs, jobs).astype(np.int64)
    for k in range(pairs):
        assert sorted(ours[k]) == list(range(jobs))
        a = p[g[f"{tag}_mp0"][k]] + lags[k]
        b = p[g[f"{tag}_mp1"][k]] + lags[k]
        key = lambda j: (0, a[j]) if a[j] < b[j] else (1, -b[j])  # noqa: E731
        assert [key(j) for j in ours[k]] == [key(j) for j in ref[k]]


@pytest.mark.parametrize("tag", SHAPE_TAGS)
def test_bounds_from_ptimes_match_reference(shapes, tag):
    """the oracle's lb1 / lb1_d / lb2 (every incumbent of the fixture) on these tables = the reference's, and lb1_d of
    the root with the Chapel min_heads = the reference built with the Chapel statement"""
    g = shapes
    parents = shape_parents(g, tag)
    for heads_mode in (0, 1):  # min_heads is never read when limit1 >= 0
        t = shape_tables(g, tag, heads_mode)
        np.testing.assert_array_equal(shape_evaluate(t, 1, parents, INT_MAX), g[f"{tag}_lb1"])
        np.testing.assert_array_equal(shape_evaluate(t, 0, parents, INT_MAX), g[f"{tag}_lb1_d"])
        for i, best in enumerate(g[f"{tag}_lb2_bests"] if t.pairs else ()):
            np.testing.assert_array_equal(shape_evaluate(t, 2, parents, int(best)), g[f"{tag}_lb2"][i],
                                          err_msg=f"lb2 best={best}")
    if f"{tag}_root_lb1_d" in g:
        t = shape_tables(g, tag, 0)
        root = np.zeros(1, dtype=po.PFSP_NODE_DTYPE)
        root["limit1"] = -1
        root["prmu"][0, : t.jobs] = np.arange(t.jobs)
        np.testing.assert_array_equal(shape_evaluate(t, 0, root, INT_MAX), g[f"{tag}_root_lb1_d"])

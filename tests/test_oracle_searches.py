"""The oracle's per-task counts and part searches (or_*_search_offload_part), on the CPU: the parts of a D-way split
add up to the whole search wherever the counts cannot depend on the order of the work (N-Queens, PFSP with ub = 1),
and each part is what its share of the warm-up pool gives when explored on its own."""
import ctypes as C

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po


def static_split(nodes, D):
    """the reference's strided split of the warm-up pool (nqueens_multigpu_chpl.chpl:199-226): task g takes
    nodes g, g + D, ...; the last task also takes the remainder"""
    n = len(nodes)
    c = n // D
    out = [nodes[g: D * c: D] for g in range(D)]
    out[-1] = np.concatenate([out[-1], nodes[D * c:]])
    return out


def subtree(N, nodes):
    tree, sol = C.c_uint64(0), C.c_uint64(0)
    nodes = np.ascontiguousarray(nodes).view(po.NQ_NODE_DTYPE)
    po.lib().or_nq_search_from(N, 1, nodes.ctypes.data, len(nodes), C.byref(tree), C.byref(sol))
    return tree.value, sol.value


@pytest.mark.parametrize("N", [9, 10, 11])
@pytest.mark.parametrize("D", [1, 2, 3, 5])
@pytest.mark.parametrize("warm_per_task", [25, 100])
def test_nq_parts_add_up_to_the_whole_search(N, D, warm_per_task):
    m, M = 25, 300
    whole = po.nq_search_offload(N, 1, m, M, D)
    assert sum(whole.task_tree[D:]) == 0
    warm = D * warm_per_task
    nodes, tree1, sol1 = tsb200.nqueens_warmup(N, warm)
    shares = static_split(nodes, D)
    parts = [po.nq_search_offload_part(N, 1, m, M, D, p, warm) for p in range(D)]
    assert (sum(p.tree for p in parts), sum(p.sol for p in parts)) == (whole.tree, whole.sol)
    for p, (r, share) in enumerate(zip(parts, shares)):
        t, s = subtree(N, share)
        # step 1 goes to part 0; step 2 and 3 of a part explore exactly the subtrees below its share
        assert (r.tree, r.sol) == (t + (tree1 if p == 0 else 0), s + (sol1 if p == 0 else 0))
        assert r.task_tree[p] <= t and all(r.task_tree[q] == 0 for q in range(8) if q != p)
    if warm_per_task == m:  # the same warm-up and split as the whole search: the same step 2 per task
        assert [p.task_tree[i] for i, p in enumerate(parts)] == list(whole.task_tree[:D])
        assert [p.task_sol[i] for i, p in enumerate(parts)] == list(whole.task_sol[:D])
        assert sum(p.offloads for p in parts) == whole.offloads


def test_nq_step_accounting():
    """tree = step 1 + the tasks' step 2 + step 3, where step 3 explores what step 2 leaves"""
    N, m, M, D = 11, 25, 300, 3
    r = po.nq_search_offload(N, 1, m, M, D)
    _, tree1, sol1 = tsb200.nqueens_warmup(N, D * m)
    step3 = r.tree - tree1 - sum(r.task_tree[:D])
    assert 0 < step3 < r.tree
    # D = 1 with chunks as large as the pool: step 2 explores everything below the warm-up pool
    one = po.nq_search_offload(N, 1, 1, 1 << 20, 1)
    _, tree1, sol1 = tsb200.nqueens_warmup(N, 1)
    assert (one.task_tree[0] + tree1, one.task_sol[0] + sol1) == (one.tree, one.sol)


def test_pfsp_parts_with_a_known_optimum():
    """ub = 1: best is the optimum throughout, so the parts add up to the whole search and every task's step 2 is
    the same whether the task runs alone or in the whole search"""
    lb, M, D = po_lb("lb1_d"), 3000, 2
    whole = po.pfsp_search_offload(14, lb, 1, 25, M, D)
    parts = [po.pfsp_search_offload_part(14, lb, 1, 25, M, D, p) for p in range(D)]
    assert (sum(p.tree for p in parts), sum(p.sol for p in parts)) == (whole.tree, whole.sol)
    assert sum(p.offloads for p in parts) == whole.offloads
    assert [p.task_tree[i] for i, p in enumerate(parts)] == list(whole.task_tree[:D])
    assert whole.best == 1377 and all(p.best == 1377 for p in parts) and list(whole.task_best[:D]) == [1377] * D
    assert sum(whole.task_tree[:D]) < whole.tree


def test_part_arguments():
    for D, part in ((2, 2), (2, -1), (9, 0), (0, 0)):
        with pytest.raises(ValueError):
            po.pfsp_search_offload_part(14, 1, 1, 25, 3000, D, part)
        with pytest.raises(ValueError):
            po.nq_search_offload_part(8, 1, 25, 300, D, part)


def po_lb(name):
    return tsb200.LB_NAMES[name]

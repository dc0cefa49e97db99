"""Generates tests/golden/nqueens_wide.json: explored tree and solutions of chosen N = 21..24 subtrees, counted by the
reference's own sequential search (baselines/nqueens/nqueens_c.c: popBack + decompose) built with MAX_QUEENS 24
(oracle/_ref/libref_nqueens24.so, oracle/queens24.mk), and the published solution totals of the whole boards.

A subtree is given by its prefix: the columns of the queens on rows 0..d-1.  Its root is the node the search creates
for that prefix (each placement swaps the chosen value into board[depth], as decompose does), so it is a node the
device pool admits.  Run from the repository root after build():  python tests/golden/make_golden_nq_wide.py
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pyoracle24 as po24  # noqa: E402

# OEIS A000170: number of ways to place N non-attacking queens on an N x N board
SOLUTIONS = {21: 314666222712, 22: 2691008701644, 23: 24233937684440, 24: 227514171973736}

# prefixes chosen so that every subtree holds 10^5 .. 10^8 nodes (greedy placements: the first safe column from 0,
# resp. from N // 2, on every row)
PREFIXES = {
    21: [[0, 2, 4, 1, 3], [10, 12, 14, 11, 13]],
    22: [[0, 2, 4, 1, 3], [11, 13, 15, 12, 14, 19]],
    23: [[0, 2, 4, 1, 3, 8, 10], [11, 13, 15, 12, 14, 19, 21]],
    24: [[0, 2, 4, 1, 3, 8, 10, 12], [12, 14, 16, 13, 15, 20, 22, 0]],
}


def subtree_root(N, prefix):
    """the node decompose creates when it places the queens of `prefix` on rows 0, 1, ... in turn"""
    node = np.zeros(1, dtype=po24.NQ_NODE_DTYPE)
    b = node["board"][0]
    b[:N] = np.arange(N)
    for d, col in enumerate(prefix):
        for i in range(d):  # isSafe: no placed queen on a diagonal of (d, col)
            assert b[i] != col - (d - i) and b[i] != col + (d - i), (N, prefix, d)
        j = int(np.nonzero(b[:N] == col)[0][0])
        assert j >= d
        b[d], b[j] = b[j], b[d]
    node["depth"] = len(prefix)
    return node


def main():
    assert po24.ref_available(), "build() first: oracle/_ref/libref_nqueens24.so is the reference's MAX_QUEENS 24 build"
    out = {"source": "reference baselines/nqueens/nqueens_c.c decompose built with MAX_QUEENS 24 (oracle/queens24.mk)",
           "solutions_oeis_a000170": {str(k): v for k, v in SOLUTIONS.items()}, "subtrees": []}
    for N, prefixes in PREFIXES.items():
        for prefix in prefixes:
            node = subtree_root(N, prefix)
            t0 = time.time()
            tree, sol = po24.nq_search_from(N, node, use_ref=True)
            print(f"N={N} prefix={prefix}: tree {tree} sol {sol} ({time.time() - t0:.1f} s)", flush=True)
            out["subtrees"].append({"N": N, "prefix": prefix, "tree": tree, "sol": sol})
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "nqueens_wide.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("wrote", path)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Golden vectors for the PFSP bound kernels beyond the Taillard tables: synthetic processing-time matrices on every
machine count 1..20 (20 jobs) and on 3, 7 and 13 machines (50 jobs), in value classes that each aim at one kernel
route of tsb_pfsp_create (template machine count, 16-bit-lane lb1, lb2 table form, lb2 refused).  Everything is
computed by the REFERENCE's own C sources compiled into oracle/_ref (oracle/Makefile):

    make -C oracle ref && python tests/golden/make_golden_shapes.py      ->  tests/golden/pfsp_shapes.npz

Per instance `tag` (listed in `tags`):
  * `{tag}_dims` (jobs, machines, pairs), `{tag}_class`, `{tag}_p_times` (machine-major), and the tables the
    reference's fill_* produce from that matrix: `_min_heads_C`, `_min_tails`, `_lags`, `_johnson_qsort`, `_mp0`,
    `_mp1`; `_min_heads_chapel` from the build with the Chapel min_heads statement (libref_pfsp_chapel.so, 20 jobs);
  * class "rs" (rising tails) overwrites min_tails after fill_* with a sequence that is not non-increasing (no
    matrix produces that; the bound functions take it as data): `_min_tails` is then the overwritten sequence and
    `_tails_set` is 1;
  * `_route`: the tsb_pfsp_route value the documented selection rules give for the tables a handle is created from
    (the oracle's fill_* with the Chapel min_heads; route_of below);
  * `_parents`: seeded nodes of every depth; `_lb1`, `_lb1_d`: the reference's bounds (slot by slot as its
    decompose_* does, ref_batch.c); `_lb2_bests` and `_lb2[i]`: lb2 at each of those incumbents — INT_MAX, values
    taken from the instance's own INT_MAX bounds (exact, +1, -1, at three quantiles) and a negative one.  Bounds
    are stored for the live slots only (k >= limit1 + 1, row-major);
  * `_root_lb1_d` (20 jobs): lb1_d of the root (limit1 = -1, the only node that reads min_heads) computed by the
    build with the Chapel min_heads statement.
Class and expected route of each instance:
  tl  p in 1..99 (Taillard-like)        every machine count; 16-bit lanes, lb2 (one-word table up to 10 machines)
  pk  p in 0..127 with 0s and 127s      every machine count; the top of lb2's packed 7-bit fields
  te  largest min_tails = 2047 / 2048    18 and 20 machines; lb2 packed (2047) / refused (2048)
  se  sum(p) + max heads + max tails = 65535 / 65536, 1 and 2 machines; 16-bit lanes at their top / scalar lb1
  wd  p up to 2^20                       scalar lb1, lb2 refused
  hv  p in 100..127                      12, 17, 20 machines (20 machines: min_tails > 2047, lb2 refused)
  rs  rising min_tails, p in 1..99       scalar lb1 with lb2 on the packed table
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pyoracle as po  # noqa: E402
from oracle import pyoracle50 as po50  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pfsp_shapes.npz")
INT_MAX = 2**31 - 1
FILL = -0x32323233
# tsb_pfsp_route bits (include/tsb200.h)
ROUTE_SIMD16, ROUTE_LB2, ROUTE_LB2U = 0x100, 0x200, 0x400


def route_of(t, wide=False):
    """the kernel route tsb_pfsp_create (wide: tsb_pfsp_create_wide) documents for tables `t`"""
    J, M, P = t.jobs, t.machines, t.pairs
    p = t.arr("p_times", J * M).reshape(M, J).astype(np.int64)
    heads, tails = t.arr("min_heads", M).astype(np.int64), t.arr("min_tails", M).astype(np.int64)
    lags = t.arr("lags", P * J).reshape(P, J) if P else np.zeros((0, J), np.int32)
    mt = 5 if M <= 5 else 10 if M <= 10 else 20
    simd16 = (not wide and (p >= 0).all() and (heads >= 0).all() and (tails >= 0).all()
              and (np.diff(tails) <= 0).all() and p.sum() + max(0, heads.max()) + max(0, tails.max()) < 65536)
    paired = sorted(set(t.arr("mp0", P)) | set(t.arr("mp1", P)))
    lb2 = (P > 0 and ((p[paired] >= 0) & (p[paired] <= 127)).all() and (lags >= 0).all()
           and (lags <= (4095 if wide else 8191)).all() and ((tails[paired] >= 0) & (tails[paired] <= 2047)).all())
    lb2u = lb2 and simd16 and mt <= 10 and P <= 45
    return mt | (ROUTE_SIMD16 if simd16 else 0) | (ROUTE_LB2 if lb2 else 0) | (ROUTE_LB2U if lb2u else 0)


def random_nodes(jobs, count, dtype, rng):
    nodes = np.zeros(count, dtype=dtype)
    for i in range(count):
        depth = 1 + i % (jobs - 1)  # 1 .. jobs-1
        nodes["depth"][i] = depth
        nodes["limit1"][i] = depth - 1
        nodes["prmu"][i, :jobs] = rng.permutation(jobs).astype(np.int32)
    return nodes


def adjust_to(p, target, measure):
    """add to p[0][0] (read by neither the Chapel min_heads, which are the last job's heads, nor min_tails) so that
    measure(p) == target"""
    p[0, 0] += target - measure(p)
    assert p[0, 0] >= 0 and measure(p) == target
    return p


def matrix(cls, J, M, rng, arg=None):
    if cls == "tl" or cls == "rs":
        return rng.integers(1, 100, size=(M, J))
    if cls == "pk":
        p = rng.integers(0, 128, size=(M, J))
        flat = p.reshape(-1)
        pick = rng.permutation(flat.size)
        n = max(2, flat.size // 12)
        flat[pick[:n]], flat[pick[n: 2 * n]] = 0, 127
        return p
    if cls == "wd":
        return rng.integers(0, 1 << 20, size=(M, J))
    if cls == "hv":
        return rng.integers(100, 128, size=(M, J))
    if cls == "te":  # job 0's tail path (machines 1..M-1) sums to `arg`, every other job's is heavier
        p = rng.integers(0, 128, size=(M, J))
        lo = -(-(arg + 1) // (M - 1))  # every other job: each of its M-1 tail values >= lo, so its sum > arg
        p[1:, 1:] = rng.integers(lo, 128, size=(M - 1, J - 1))
        q, r = divmod(arg, M - 1)
        p[1:, 0] = q + (np.arange(M - 1) < r)
        return p
    if cls == "se":  # sum(p) + max Chapel min_heads + max min_tails == arg
        p = rng.integers(arg // (J * M) - 300, arg // (J * M) - 100, size=(M, J))

        def measure(q):
            t = po.tables_from_ptimes(q, heads_mode=0)
            return int(q.sum()) + max(t.arr("min_heads", M)) + max(t.arr("min_tails", M))
        return adjust_to(p, arg, measure)
    raise ValueError(cls)


def ref_data(L, p, tails=None):
    """(lb1*, lb2*) of the reference for matrix p[M, J], built by its own fill_* (pfsp_c.c:236-246 with the Taillard
    generator replaced by p); `tails` overwrites min_tails afterwards"""
    M, J = p.shape
    d1 = L.new_bound_data(J, M)
    np.ctypeslib.as_array(d1.contents.p_times, shape=(M * J,))[:] = p.reshape(-1)
    L.fill_min_heads_tails(d1)
    if tails is not None:
        np.ctypeslib.as_array(d1.contents.min_tails, shape=(M,))[:] = tails
    d2 = L.new_johnson_bd_data(d1)
    L.fill_machine_pairs(d2)
    L.fill_lags(d1.contents.p_times, d2)
    L.fill_johnson_schedules(d1.contents.p_times, d2)
    return d1, d2


def ref_bounds(L, d1, d2, kind, nodes, best):
    """the live slots (k >= limit1 + 1, row-major) of the bounds the reference computes for `nodes`"""
    jobs = d1.contents.nb_jobs
    out = np.full(nodes.shape[0] * jobs, FILL, dtype=np.int32)
    L.ref_pfsp_evaluate_range(d1, d2, kind, nodes.ctypes.data_as(C.c_void_p), 0, nodes.shape[0], int(best),
                              out.ctypes.data_as(C.c_void_p))
    live = np.arange(jobs)[None, :] >= (nodes["limit1"][:, None].astype(np.int64) + 1)
    return out.reshape(-1, jobs)[live]


def lb2_bests(inf):
    vals = np.sort(inf)
    bests = [INT_MAX]
    for q in (0.1, 0.5, 0.9):
        v = int(vals[int(q * (vals.size - 1))])
        bests += [v, v + 1, v - 1]
    bests.append(-1)
    return np.array(list(dict.fromkeys(bests)), dtype=np.int64)


def add_instance(out, tags, tag, cls, p, rng, jobs50=False, tails=None):
    M, J = p.shape
    p = p.astype(np.int32)
    L = po.ref_pfsp_named("50") if jobs50 else po.ref_pfsp()
    d1, d2 = ref_data(L, p, tails)
    pairs = d2.contents.nb_machine_pairs
    asarr = lambda ptr, n: np.ctypeslib.as_array(ptr, shape=(n,)).astype(np.int32).copy() if n else np.zeros(0, np.int32)  # noqa: E731
    out[f"{tag}_dims"] = np.array([J, M, pairs], dtype=np.int32)
    out[f"{tag}_class"] = np.array(cls)
    out[f"{tag}_p_times"] = p.reshape(-1).copy()
    out[f"{tag}_min_heads_C"] = asarr(d1.contents.min_heads, M)
    out[f"{tag}_min_tails"] = asarr(d1.contents.min_tails, M)
    out[f"{tag}_tails_set"] = np.array([tails is not None], dtype=np.int32)
    lags = asarr(d2.contents.lags, pairs * J)
    out[f"{tag}_lags"] = lags.astype(np.int16) if lags.size == 0 or lags.max() < 2**15 else lags  # (smaller file)
    out[f"{tag}_johnson_qsort"] = asarr(d2.contents.johnson_schedules, pairs * J).astype(np.uint8)
    out[f"{tag}_mp0"] = asarr(d2.contents.machine_pairs_1, pairs)
    out[f"{tag}_mp1"] = asarr(d2.contents.machine_pairs_2, pairs)
    mod = po50 if jobs50 else po
    t = mod.tables_from_ptimes(p, heads_mode=0)
    if tails is not None:
        np.ctypeslib.as_array(t.min_tails)[:M] = tails
    out[f"{tag}_route"] = np.array([route_of(t, wide=jobs50)], dtype=np.int32)
    nodes = random_nodes(J, J - 1 if jobs50 else 40, mod.PFSP_NODE_DTYPE, rng)
    out[f"{tag}_parents"] = nodes.view(np.uint8).reshape(-1)
    out[f"{tag}_lb1"] = ref_bounds(L, d1, d2, 1, nodes, INT_MAX)
    out[f"{tag}_lb1_d"] = ref_bounds(L, d1, d2, 0, nodes, INT_MAX)
    if pairs:
        bests = lb2_bests(ref_bounds(L, d1, d2, 2, nodes, INT_MAX))
        out[f"{tag}_lb2_bests"] = bests
        out[f"{tag}_lb2"] = np.stack([ref_bounds(L, d1, d2, 2, nodes, b) for b in bests])
    if not jobs50:
        Lc = po.ref_pfsp(chapel_heads=True)
        c1, c2 = ref_data(Lc, p, tails)
        out[f"{tag}_min_heads_chapel"] = asarr(c1.contents.min_heads, M)
        root = np.zeros(1, dtype=po.PFSP_NODE_DTYPE)
        root["limit1"] = -1
        root["prmu"][0, :J] = np.arange(J)
        out[f"{tag}_root_lb1_d"] = ref_bounds(Lc, c1, c2, 0, root, INT_MAX)
    tags.append(tag)


def main():
    rng = np.random.default_rng(0x5A9E)
    out, tags = {}, []
    J = 20
    for cls in ("tl", "pk"):
        for M in range(1, 21):
            add_instance(out, tags, f"j20_{cls}_m{M:02d}", cls, matrix(cls, J, M, rng), rng)
    for M in (18, 20):
        for target in (2047, 2048):
            add_instance(out, tags, f"j20_te{target}_m{M:02d}", "te", matrix("te", J, M, rng, target), rng)
    for M in (1, 2):
        for target in (65535, 65536):
            add_instance(out, tags, f"j20_se{target}_m{M:02d}", "se", matrix("se", J, M, rng, target), rng)
    for M in (3, 7, 13, 20):
        add_instance(out, tags, f"j20_wd_m{M:02d}", "wd", matrix("wd", J, M, rng), rng)
    for M in (12, 17, 20):
        add_instance(out, tags, f"j20_hv_m{M:02d}", "hv", matrix("hv", J, M, rng), rng)
    for M in (4, 7, 13):
        tails = rng.integers(0, 400, size=M).astype(np.int32)
        tails[1] = tails[0] + 37  # rises at least once
        add_instance(out, tags, f"j20_rs_m{M:02d}", "rs", matrix("rs", J, M, rng), rng, tails=tails)
    J = 50
    for cls, M in (("tl", 3), ("tl", 7), ("tl", 13), ("pk", 7), ("wd", 13)):
        add_instance(out, tags, f"j50_{cls}_m{M:02d}", cls, matrix(cls, J, M, rng), rng, jobs50=True)
    out["tags"] = np.array(tags)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(tags), "instances;", os.path.getsize(OUT), "bytes")
    for tag in tags:
        r = int(out[f"{tag}_route"][0])
        print(f"  {tag:18s} mt={r & 0xFF:2d} simd16={int(bool(r & ROUTE_SIMD16))} lb2={int(bool(r & ROUTE_LB2))} "
              f"lb2u={int(bool(r & ROUTE_LB2U))}")


if __name__ == "__main__":
    main()

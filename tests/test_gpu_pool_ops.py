"""Both device pools (the PFSP and N-Queens handles' DevicePool: extents, 2-record alignment for PFSP, compaction,
growth, the stack a persistent launch needs) under any order of operations, against a host model of the reference's
Pool (lib/commons/Pool.chpl, Pool_par.chpl):
  push       pushBack of every node, in order;
  round      popBackBulk(m, M) (nothing below m nodes) -> the oracle's evaluate + generate_children (po.pfsp_expand /
             po.nq_expand) -> the children pushed;
  steal      popFrontBulkFree: size // 2 nodes from the front, only when size >= 2 m, to the top of the thief;
  drain      every node, oldest first.
pool_step, pool_run (inside and outside the persistent kernels), pool_steal and pool_drain are checked node for node.
The GPU tests are marked one by one: the model's own check runs without a GPU."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import tsb200
from oracle import pyoracle as po
from test_gpu_parity import rand_nq, rand_pfsp
from tsb200 import _lib

OPT14 = 1377
INT64_MAX = 2**63 - 1
PFR_MAX_M = 20000  # pfsp_rounds.cuh: the largest M pool_run takes the persistent PFSP kernel for
SMALL_CAP = 2000   # TSB200_POOL_CAP of half the operation sequences


@pytest.fixture(autouse=True)
def default_env(monkeypatch):
    for v in ("TSB200_NO_SIMD16", "TSB200_NO_ROUNDS", "TSB200_POOL_CAP"):
        monkeypatch.delenv(v, raising=False)


def sm_count():
    n = int(tsb200.lib().tsb_device_sm_count(0))
    assert n > 0
    return n


def nq_one_pool_capacity(sms):
    """ll_tiers.h ll_pool_capacity for one pool: the largest M one pool's persistent N-Queens kernel takes"""
    return min(sms, 256) * 512


# ------------------------------------------------------------------------------------------ the host model
class PfspProblem:
    name, fanout = "pfsp", 20
    dtype, odtype = tsb200.PFSP_NODE_DTYPE, po.PFSP_NODE_DTYPE

    def __init__(self, lb, best=OPT14, inst=14):
        self.inst, self.lb, self.best0 = inst, lb, best
        self.frontier = None
        self.t = po.tables(inst, heads_mode=0)

    def expand(self, chunk, best):
        kids, sol, after = po.pfsp_expand(self.t, tsb200.LB_NAMES[self.lb], chunk.view(self.odtype), best)
        return kids.view(self.dtype), sol, after

    def handle(self, M):
        return tsb200.PfspEvaluator(self.inst, M=M)

    def nodes(self, rng, count):
        """deep random nodes without an incumbent (nothing is pruned); with the optimum, nodes of the search tree
        (random ones rarely have a child there): depth-2 and depth-3 descendants of the root"""
        if self.best0 == INT64_MAX:
            return rand_pfsp(rng, 20, count, depth_lo=13)
        if self.frontier is None:
            root = np.zeros(1, dtype=self.dtype)
            root["limit1"] = -1
            root["prmu"][0] = np.arange(20)
            d1, _, _ = self.expand(root, self.best0)
            d2, _, _ = self.expand(d1, self.best0)
            d3, _, _ = self.expand(d2, self.best0)
            self.frontier = np.concatenate([d2, d3])
        return self.frontier[rng.integers(0, self.frontier.shape[0], size=count)]

    def step(self, ev, m, M, best):
        n, c, s, b = ev.pool_step(self.lb, m, M, best)
        return (n, c, s), b

    def run(self, ev, m, M, best, rounds):
        got = ev.pool_run(self.lb, m, M, best, max_rounds=rounds)
        return tuple(got[:4]), got[4]


class NqProblem:
    name = "nqueens"
    dtype, odtype = tsb200.NQ_NODE_DTYPE, po.NQ_NODE_DTYPE
    best0 = None

    def __init__(self, N):
        self.N = self.fanout = N

    def expand(self, chunk, best):
        kids, sol = po.nq_expand(chunk.view(self.odtype), self.N)
        return kids.view(self.dtype), sol, best

    def handle(self, M):
        return tsb200.NQueensEvaluator(self.N, M=M)

    def nodes(self, rng, count):
        return rand_nq(rng, self.N, count, depth_lo=max(0, self.N - 7))

    def step(self, ev, m, M, best):
        return ev.pool_step(m, M), best

    def run(self, ev, m, M, best, rounds):
        return tuple(ev.pool_run(m, M, max_rounds=rounds)), best


class ModelPool:
    """the reference's Pool of one task on the host, with the offload rounds of the oracle"""

    def __init__(self, prob):
        self.prob = prob
        self.pool = np.zeros(0, dtype=prob.dtype)
        self.best = prob.best0
        self.rounds = []

    @property
    def size(self):
        return self.pool.shape[0]

    def push(self, nodes):
        self.pool = np.concatenate([self.pool, nodes])

    def step(self, m, M):
        """one round: (parents, children, solutions); (0, 0, 0) below m nodes"""
        if self.size < m:
            return 0, 0, 0
        n = min(self.size, M)
        s0 = self.size - n
        kids, sol, self.best = self.prob.expand(np.ascontiguousarray(self.pool[s0:]), self.best)
        self.pool = np.concatenate([self.pool[:s0], kids])
        self.rounds.append((n, kids.shape[0], sol))
        return n, kids.shape[0], sol

    def run(self, m, M, max_rounds):
        tot = [0, 0, 0, 0]
        while tot[0] < max_rounds:
            n, c, s = self.step(m, M)
            if n == 0:
                break
            tot = [tot[0] + 1, tot[1] + n, tot[2] + c, tot[3] + s]
        return tuple(tot)

    def steal_to(self, thief, m):
        if self.size < 2 * m:
            return 0
        k = self.size // 2
        thief.push(self.pool[:k])
        self.pool = self.pool[k:].copy()
        return k

    def drain(self):
        out, self.pool = self.pool, np.zeros(0, dtype=self.prob.dtype)
        return out


def model_search_from_the_root(prob, root, m, M):
    """the offload loop until the pool is empty: (children, solutions, best)"""
    pool = ModelPool(prob)
    pool.push(root)
    tot = pool.run(m, M, 10**12)
    return tot[2], tot[3], pool.best


# ------------------------------------------------------------------------------------------ the model's own check
@pytest.mark.parametrize("lb,key", [("lb1", "ta014_lb1_ub1"), ("lb1_d", "ta014_lb0_ub1")])
def test_model_pfsp_loop_gives_the_reference_counts(golden_dir, lb, key):
    """the model's loop from the ta014 root (m = 1, M = 50 000, best = the optimum) explores the reference's tree"""
    want = json.load(open(os.path.join(golden_dir, "counts.json")))["pfsp"][key]
    root = np.zeros(1, dtype=tsb200.PFSP_NODE_DTYPE)
    root["limit1"] = -1
    root["prmu"][0] = np.arange(20)
    assert model_search_from_the_root(PfspProblem(lb), root, 1, 50000) == (want["tree"], want["sol"], want["best"])


def test_model_nqueens_loop_gives_the_reference_counts(golden_dir):
    want = json.load(open(os.path.join(golden_dir, "counts.json")))["nqueens"]["10"]
    root = np.zeros(1, dtype=tsb200.NQ_NODE_DTYPE)
    root["board"][0, :10] = np.arange(10)
    got = model_search_from_the_root(NqProblem(10), root, 1, 50000)
    assert got[:2] == (want["tree"], want["sol"])


def test_model_steal_takes_the_front_half():
    prob = NqProblem(8)
    a, b = ModelPool(prob), ModelPool(prob)
    nodes = rand_nq(np.random.default_rng(1), 8, 11)
    a.push(nodes)
    assert a.steal_to(b, 6) == 0 and a.steal_to(b, 5) == 5
    assert b.pool.tobytes() == nodes[:5].tobytes() and a.pool.tobytes() == nodes[5:].tobytes()


# ------------------------------------------------------------------------------------------ random sequences
def check_drain(ev, model, push_back=True):
    got = ev.pool_drain()
    want = model.drain()
    assert ev.pool_size == 0 and got.tobytes() == np.ascontiguousarray(want).tobytes()
    if push_back and got.shape[0]:
        ev.pool_push(got)
        model.push(got)


def make_problem(problem, seed):
    if problem == "pfsp":
        return PfspProblem(("lb1", "lb1_d")[seed % 2], (OPT14, INT64_MAX)[seed // 2 % 2])
    return NqProblem((8, 12)[seed % 2])


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("problem", ["pfsp", "nqueens"])
def test_random_operation_sequences(problem, seed, monkeypatch):
    """60 random operations on two handles: pushes of 0, 1, an odd number and thousands of nodes, pool_step,
    pool_run of a few rounds inside and outside the persistent kernel, steals either way (moving nodes or not),
    drains with the nodes pushed back; with a 2000-record arena for half of the seeds"""
    small = seed >= 4
    if small:
        monkeypatch.setenv("TSB200_POOL_CAP", str(SMALL_CAP))
    prob = make_problem(problem, seed)
    rng = np.random.default_rng(11200 + 100 * (problem == "pfsp") + seed)
    if problem == "pfsp":
        inside, outside = PFR_MAX_M, PFR_MAX_M + 1
    else:
        inside = nq_one_pool_capacity(sm_count())
        outside = inside + 1
    models = [ModelPool(prob), ModelPool(prob)]
    bests = [prob.best0, prob.best0]
    # a persistent launch on a pool of several extents, or of one that does not start at position 0, compacts it
    # first (DevicePool::make_stack); `scattered` marks the pools a step or a steal left so.  It compacts within the
    # arena it has when the launch's worst case fits that arena, whose size is at least `cap_lo`: the initial
    # capacity, and every pool size and every round's worst case the handle has had room for
    scattered = [False, False]
    cap_lo = [SMALL_CAP if small else 1 << 20] * 2
    launches_on_scattered, max_size = 0, 0
    ops = []
    with prob.handle(outside) as e0, prob.handle(outside) as e1:
        evs = [e0, e1]
        for _ in range(60):
            op = rng.choice(["push", "push", "step", "run", "run", "run", "steal", "steal", "drain"])
            i = int(rng.integers(2))
            if op == "run" and any(scattered) and rng.random() < 0.5:
                i = scattered.index(True) if not all(scattered) else i
            ev, mod = evs[i], models[i]
            if op == "push":
                k = int(rng.choice([0, 1, 37, 3001]))
                nodes = prob.nodes(rng, k)
                ev.pool_push(nodes)
                mod.push(nodes)
            elif op == "step":
                m, M = int(rng.choice([1, 25])), int(rng.choice([300, 5000]))
                if mod.size >= m:
                    cap_lo[i] = max(cap_lo[i], mod.size + min(mod.size, M) * prob.fanout)
                got, bests[i] = prob.step(ev, m, M, bests[i])
                assert got == mod.step(m, M) and bests[i] == mod.best
                scattered[i] |= got[1] > 0
            elif op == "run":
                m, M, k = int(rng.choice([1, 25])), int(rng.choice([inside, inside, outside])), int(rng.integers(1, 4))
                size, need = mod.size, None
                if size >= m:
                    n = min(size, M)
                    need = size - n + n * prob.fanout
                r0 = len(mod.rounds)
                got, bests[i] = prob.run(ev, m, M, bests[i], k)
                assert got == mod.run(m, M, k) and bests[i] == mod.best
                if M == outside:
                    scattered[i] |= any(c > 0 for _, c, _ in mod.rounds[r0:])
                elif need is not None:
                    launches_on_scattered += scattered[i] and need <= cap_lo[i]
                    scattered[i] = False  # (or scattered again by a round redone by pool_step: not counted)
                    cap_lo[i] = max(cap_lo[i], need)
            elif op == "steal":
                v = 1 - i
                m = int(rng.choice([1, 25, models[v].size // 2 + 1]))
                had = mod.size
                want = models[v].steal_to(mod, m)
                assert ev.pool_steal_from(evs[v], m) == want
                if want:  # the victim's front moved; the thief's stolen nodes are an extent above its own
                    scattered[v] = True
                    scattered[i] |= had > 0
            else:
                check_drain(ev, mod)
                scattered[i] = False
            ops.append(op)
            for j, (e, mo) in enumerate(zip(evs, models)):
                assert e.pool_size == mo.size, (len(ops), ops[-1])
                cap_lo[j] = max(cap_lo[j], mo.size)
            max_size = max(max_size, models[0].size, models[1].size)
        for ev, mod in zip(evs, models):
            check_drain(ev, mod, push_back=False)
    assert {"push", "step", "run", "steal", "drain"} <= set(ops)
    assert launches_on_scattered > 0  # a compaction inside the arena it had
    if small:
        assert max_size > SMALL_CAP  # the arena grew


# ------------------------------------------------------------------------------------------ PFSP steal, byte level
@pytest.mark.gpu
def test_pfsp_steal_moves_the_oldest_half_in_order():
    """the PFSP twin of test_pool_steal_moves_the_oldest_half_in_order: 1001 + 7 nodes moves 500 (501 / 507 left);
    size = 2 m moves m, size = 2 m - 1 nothing"""
    m = 25
    rng = np.random.default_rng(12)
    nodes = rand_pfsp(rng, 20, 1001, depth_lo=12)
    own = rand_pfsp(rng, 20, 7, depth_lo=12)
    with tsb200.PfspEvaluator(14, M=5000) as victim, tsb200.PfspEvaluator(14, M=5000) as thief:
        victim.pool_push(nodes)
        thief.pool_push(own)
        assert thief.pool_steal_from(victim, m) == 500
        assert (victim.pool_size, thief.pool_size) == (501, 507)
        assert thief.pool_steal_from(victim, 251) == 0 and victim.pool_size == 501
        assert thief.pool_drain().tobytes() == np.concatenate([own, nodes[:500]]).tobytes()
        assert victim.pool_drain().tobytes() == np.ascontiguousarray(nodes[500:]).tobytes()
        for size, moved in ((2 * m, m), (2 * m - 1, 0)):
            victim.pool_push(nodes[:size])
            assert thief.pool_steal_from(victim, m) == moved
            assert (victim.pool_size, thief.pool_size) == (size - moved, moved)
            assert thief.pool_drain().tobytes() == nodes[:moved].tobytes()
            assert victim.pool_drain().tobytes() == nodes[moved:size].tobytes()


def run_to_exhaustion(ev):
    got = ev.pool_run("lb1", 1, 5000, OPT14)
    assert ev.pool_size == 0 and got[4] == OPT14
    return got[2], got[3]


@pytest.mark.gpu
@pytest.mark.parametrize("victim_kind", ["stack_from_pool_run", "many_extents_from_pool_steps"])
@pytest.mark.parametrize("thief_kind", ["no_arena", "aligned_top_overflows"])
def test_pfsp_steal_across_extents_and_arenas(victim_kind, thief_kind, monkeypatch):
    """the victim: the stack a persistent launch left, or a pool of more than EXP_MAX_PIECES (8) extents after
    pool_step rounds, so that the stolen half spans several extents; the thief: a handle that never allocated an
    arena, or one whose aligned top plus the stolen half passes the end of its arena.  Both pools are compared node
    for node and keep running: their trees add up to the tree of the pool before the steal"""
    prob = PfspProblem("lb1", OPT14)
    rng = np.random.default_rng(13 + 2 * (victim_kind[0] == "s") + (thief_kind[0] == "n"))
    vm, tm = ModelPool(prob), ModelPool(prob)
    with tsb200.PfspEvaluator(14, M=5000) as victim, tsb200.PfspEvaluator(14, M=5000) as thief:
        if victim_kind == "stack_from_pool_run":
            # depth 16 / 17 without an incumbent: two rounds with children and without leaves, both in the kernel
            start = rand_pfsp(rng, 20, 200, depth_lo=16)
            start["depth"][:] = np.minimum(start["depth"], 17)
            start["limit1"][:] = start["depth"] - 1
            victim.pool_push(start)
            vm.push(start)
            vm.best = INT64_MAX
            got, _ = prob.run(victim, 25, 5000, vm.best, 2)
            assert got == vm.run(25, 5000, 2) and got[0] == 2 and vm.size > 0
        else:
            # 11 nodes with many children, then rounds of 10 parents: each round leaves part of the previous round's
            # children below it and adds an extent
            start = rand_pfsp(rng, 20, 11, depth_lo=2)
            start["depth"][:] = np.minimum(start["depth"], 5)
            start["limit1"][:] = start["depth"] - 1
            victim.pool_push(start)
            vm.push(start)
            vm.best = INT64_MAX
            for _ in range(10):
                got, _ = prob.step(victim, 1, 10, vm.best)
                assert got == vm.step(1, 10)
            kids = [c for _, c, _ in vm.rounds]
            assert all(c > 10 for c in kids[:-1])  # every round's chunk lies inside the previous round's children
            assert len(kids) + 1 > 8  # extents: the start's remainder and one per round
        if thief_kind == "aligned_top_overflows":
            # the stolen half `want` odd and >= 1025, the thief's own k = 2000 - want nodes odd: its top + want fills
            # its 2000-record arena exactly, its aligned top (k + 1) + want is one past the end
            want = max(1025, vm.size // 2)
            want += 1 - want % 2
            more = rand_pfsp(rng, 20, max(0, 2 * want - vm.size), depth_lo=15)
            victim.pool_push(more)  # (onto the top extent: the victim's layout stays what it was)
            vm.push(more)
            assert vm.size // 2 == want and vm.size < 4000
            k = SMALL_CAP - want
            assert k % 2 and k + 1024 <= SMALL_CAP
            # (TSB200_POOL_CAP is read when an arena is first allocated: only the thief's is small)
            monkeypatch.setenv("TSB200_POOL_CAP", str(SMALL_CAP))
            own = rand_pfsp(rng, 20, k, depth_lo=15)
            thief.pool_push(own)
            tm.push(own)
            monkeypatch.delenv("TSB200_POOL_CAP")
        want = vm.steal_to(tm, 25)
        assert thief.pool_steal_from(victim, 25) == want > 0
        assert (victim.pool_size, thief.pool_size) == (vm.size, tm.size)
        both = np.concatenate([tm.pool, vm.pool])
        check_drain(victim, vm)
        check_drain(thief, tm)
        a, b = run_to_exhaustion(victim), run_to_exhaustion(thief)
    with tsb200.PfspEvaluator(14, M=5000) as one:
        one.pool_push(both)
        c = run_to_exhaustion(one)
    assert (a[0] + b[0], a[1] + b[1]) == c


# ------------------------------------------------------------------------------------------ drain, too small
@pytest.mark.gpu
@pytest.mark.parametrize("problem", ["pfsp", "nqueens"])
def test_pool_drain_with_one_record_too_few(problem):
    """capacity size - 1: TSB_ENOMEM, *n = size, and the pool as it was (after a persistent launch: for N-Queens the
    pool then lives in the kernel's own format)"""
    prob = PfspProblem("lb1", INT64_MAX) if problem == "pfsp" else NqProblem(12)
    rng = np.random.default_rng(14)
    mod = ModelPool(prob)
    L = tsb200.lib()
    drain = L.tsb_pfsp_pool_drain if problem == "pfsp" else L.tsb_nq_pool_drain
    with prob.handle(5000) as ev:
        start = prob.nodes(rng, 301)
        ev.pool_push(start)
        mod.push(start)
        got, _ = prob.run(ev, 25, 5000, mod.best, 2)
        assert got == mod.run(25, 5000, 2)
        size = mod.size
        assert size > 1
        buf = np.zeros(size, dtype=prob.dtype)
        n = C.c_int64(-7)
        assert drain(ev._h, buf.ctypes.data, size - 1, C.byref(n)) == _lib.ENOMEM
        assert n.value == size and ev.pool_size == size
        assert not buf.view(np.uint8).any()
        got, _ = prob.step(ev, 1, 300, mod.best)
        assert got == mod.step(1, 300)
        check_drain(ev, mod, push_back=False)

"""The resumable host-pool searches (tsb_nq_search_ckpt, tsb_pfsp_search_ckpt, tsb_pfsp_search_ckpt_wide) where no GPU
is needed: every argument is refused with the code of the twin (tsb_nq_search / tsb_nq_search_wide, tsb_pfsp_search,
tsb_pfsp_search_wide) before any device call and no file is written; a checkpoint of the other kind of search (host
pools: Params::pools = 0, and c = 1 for N-Queens, whose device-pool files have pools = 0 too; PFSP device pools: 1..4),
of another node width, or with a host task holding other than one pool is refused with TSB_EINVAL and left as it is."""
import ctypes as C
import os
import struct

import pytest

import tsb200
from tsb200 import _lib

NQ, PFSP = 1, 2


@pytest.fixture(scope="module")
def L():
    return tsb200.lib()


def test_declared_and_bound(L):
    for name in ("tsb_nq_search_ckpt", "tsb_pfsp_search_ckpt", "tsb_pfsp_search_ckpt_wide"):
        assert hasattr(L, name) and name in _lib.SYMBOLS


# ------------------------------------------------------------------------------------------ arguments
def nq_pair(L, path, max_queens=20, N=12, g=1, m=25, M=1000, D=1):
    """(twin, resumable form) on the same arguments"""
    st = _lib.SearchStats()
    twin = (L.tsb_nq_search(N, g, m, M, D, C.byref(st)) if max_queens == 20
            else L.tsb_nq_search_wide(max_queens, N, g, m, M, D, C.byref(st)))
    return twin, L.tsb_nq_search_ckpt(max_queens, N, g, m, M, D, os.fsencode(str(path)), 0.0, C.byref(st))


@pytest.mark.parametrize("args", [dict(N=0), dict(N=25), dict(N=-1), dict(g=0), dict(m=0), dict(M=0), dict(M=-5),
                                  dict(D=0), dict(D=9), dict(max_queens=24, N=25), dict(max_queens=24, D=9),
                                  dict(max_queens=24, g=0), dict(max_queens=24, m=0)])
def test_nq_arguments(L, tmp_path, args):
    assert nq_pair(L, tmp_path / "ck", **args) == (_lib.EINVAL, _lib.EINVAL)
    assert os.listdir(tmp_path) == []


def test_nq_max_queens_path_seconds_out(L, tmp_path):
    st = _lib.SearchStats()
    path = os.fsencode(str(tmp_path / "ck"))
    for mq in (0, 19, 21, 23, 25):  # (the twin of 24, tsb_nq_search_wide, refuses every other build as well)
        assert L.tsb_nq_search_ckpt(mq, 12, 1, 25, 1000, 1, path, 0.0, C.byref(st)) == _lib.EINVAL
        assert L.tsb_nq_search_wide(mq, 12, 1, 25, 1000, 1, C.byref(st)) == _lib.EINVAL
    assert L.tsb_nq_search_ckpt(20, 12, 1, 25, 1000, 1, None, 0.0, C.byref(st)) == _lib.EINVAL
    assert L.tsb_nq_search_ckpt(20, 12, 1, 25, 1000, 1, b"", 0.0, C.byref(st)) == _lib.EINVAL
    assert L.tsb_nq_search_ckpt(20, 12, 1, 25, 1000, 1, path, float("nan"), C.byref(st)) == _lib.EINVAL
    assert L.tsb_nq_search_ckpt(20, 12, 1, 25, 1000, 1, path, 0.0, None) == _lib.EINVAL
    assert L.tsb_nq_search_ckpt(24, 12, 1, 25, 1000, 1, path, 0.0, None) == _lib.EINVAL
    assert os.listdir(tmp_path) == []


def pfsp_pair(L, path, inst=14, lb=1, ub=1, m=25, M=1000, D=1):
    st = _lib.SearchStats()
    return (L.tsb_pfsp_search(inst, lb, ub, m, M, D, C.byref(st)),
            L.tsb_pfsp_search_ckpt(inst, lb, ub, m, M, D, os.fsencode(str(path)), 0.0, C.byref(st)))


@pytest.mark.parametrize("args,code", [
    (dict(lb=3), _lib.EINVAL), (dict(lb=-1), _lib.EINVAL), (dict(ub=2), _lib.EINVAL), (dict(ub=-1), _lib.EINVAL),
    (dict(m=0), _lib.EINVAL), (dict(M=0), _lib.EINVAL), (dict(D=0), _lib.EINVAL), (dict(D=9), _lib.EINVAL),
    (dict(inst=0), _lib.EINVAL), (dict(inst=121), _lib.EINVAL), (dict(inst=31), _lib.EUNSUPPORTED),
    (dict(inst=61), _lib.EUNSUPPORTED)])
def test_pfsp_arguments(L, tmp_path, args, code):
    assert pfsp_pair(L, tmp_path / "ck", **args) == (code, code)
    assert os.listdir(tmp_path) == []


def pfsp_wide_pair(L, path, max_jobs=50, inst=31, lb=1, ub=1, m=25, M=1000, D=1):
    st = _lib.SearchStats()
    return (L.tsb_pfsp_search_wide(max_jobs, inst, lb, ub, m, M, D, C.byref(st)),
            L.tsb_pfsp_search_ckpt_wide(max_jobs, inst, lb, ub, m, M, D, os.fsencode(str(path)), 0.0, C.byref(st)))


# (the rules of tests/test_pfsp50_search.py: max_jobs only 50, inst only 31..60, the other checks first)
@pytest.mark.parametrize("args,code", [
    (dict(max_jobs=20), _lib.EINVAL), (dict(max_jobs=49), _lib.EINVAL), (dict(max_jobs=100), _lib.EINVAL),
    (dict(lb=3), _lib.EINVAL), (dict(lb=-1), _lib.EINVAL), (dict(ub=2), _lib.EINVAL), (dict(m=0), _lib.EINVAL),
    (dict(M=0), _lib.EINVAL), (dict(D=0), _lib.EINVAL), (dict(D=9), _lib.EINVAL),
    (dict(inst=30), _lib.EUNSUPPORTED), (dict(inst=61), _lib.EUNSUPPORTED), (dict(inst=1), _lib.EUNSUPPORTED),
    (dict(inst=0), _lib.EUNSUPPORTED), (dict(inst=121), _lib.EUNSUPPORTED),
    (dict(max_jobs=20, inst=30), _lib.EINVAL), (dict(inst=14, m=0), _lib.EINVAL)])
def test_pfsp_wide_arguments(L, tmp_path, args, code):
    assert pfsp_wide_pair(L, tmp_path / "ck", **args) == (code, code)
    assert os.listdir(tmp_path) == []


def test_pfsp_path_seconds_out(L, tmp_path):
    st = _lib.SearchStats()
    path = os.fsencode(str(tmp_path / "ck"))
    for fn, pre in ((L.tsb_pfsp_search_ckpt, (14,)), (L.tsb_pfsp_search_ckpt_wide, (50, 31))):
        assert fn(*pre, 1, 1, 25, 1000, 1, None, 0.0, C.byref(st)) == _lib.EINVAL
        assert fn(*pre, 1, 1, 25, 1000, 1, b"", 0.0, C.byref(st)) == _lib.EINVAL
        assert fn(*pre, 1, 1, 25, 1000, 1, path, float("nan"), C.byref(st)) == _lib.EINVAL
        assert fn(*pre, 1, 1, 25, 1000, 1, path, 0.0, None) == _lib.EINVAL
    assert os.listdir(tmp_path) == []


def test_missing_file_without_device(L, tmp_path):
    if L.tsb_device_count() > 0:
        pytest.skip("a CUDA device is present: the search would run")
    st = _lib.SearchStats()
    path = os.fsencode(str(tmp_path / "ck"))
    assert L.tsb_nq_search_ckpt(20, 12, 1, 25, 1000, 1, path, 0.0, C.byref(st)) == _lib.ENODEV
    assert L.tsb_nq_search_ckpt(24, 12, 1, 25, 1000, 1, path, 0.0, C.byref(st)) == _lib.ENODEV
    assert L.tsb_pfsp_search_ckpt(14, 1, 1, 25, 1000, 1, path, 0.0, C.byref(st)) == _lib.ENODEV
    assert L.tsb_pfsp_search_ckpt_wide(50, 31, 1, 1, 25, 1000, 1, path, 0.0, C.byref(st)) == _lib.ENODEV
    assert os.listdir(tmp_path) == []


# ------------------------------------------------------------------------------------------ hand-built checkpoints
def checkpoint(problem, rec, a, b, c, m, M, pools, tasks):
    """a well-formed checkpoint (layout: csrc/search_ckpt.cpp) of len(tasks) tasks; tasks[i] = (finished, left nodes,
    [nodes of each pool state]), every node a zero record of `rec` bytes"""
    out = b"TSB200CK" + struct.pack("<3I7i", 1, problem, rec, a, b, c, m, M, len(tasks), pools)
    out += struct.pack("<QQqddQ", 0, 0, 2**63 - 1, 0.0, 0.0, 0)
    for finished, left, states in tasks:
        out += struct.pack("<5Qq2IQ", 0, 0, 0, 0, 0, 2**63 - 1, int(finished), len(states), left) + bytes(rec * left)
        for n in states:
            out += struct.pack("<qQ", 2**63 - 1, n) + bytes(rec * n)
    h = 0xcbf29ce484222325
    for i in range(0, len(out) - len(out) % 8, 8):
        h = ((h ^ int.from_bytes(out[i:i + 8], "little")) * 0x100000001b3) & (2**64 - 1)
    for x in out[len(out) - len(out) % 8:]:
        h = ((h ^ x) * 0x100000001b3) & (2**64 - 1)
    return out + struct.pack("<Q", h ^ (h >> 29))


M_, m_ = 64, 5
ONE_TASK = [(False, 0, [3])]


def nq_host(rec=21, tasks=ONE_TASK):  # N = 12, g = 1; c = 1 marks N-Queens host pools
    return checkpoint(NQ, rec, 12, 1, 1, m_, M_, 0, tasks)


def nq_device(rec=21, tasks=ONE_TASK):
    return checkpoint(NQ, rec, 12, 1, 0, m_, M_, 0, tasks)


def pf_host(rec=88, inst=14, tasks=ONE_TASK):  # lb1, ub 0
    return checkpoint(PFSP, rec, inst, 1, 0, m_, M_, 0, tasks)


def pf_device(rec=88, inst=14, pools=1, tasks=ONE_TASK):
    return checkpoint(PFSP, rec, inst, 1, 0, m_, M_, pools, tasks)


def calls(L, path, D=1):
    """every resumable search on the parameters of the hand-built files, by name"""
    st = _lib.SearchStats()
    p = os.fsencode(str(path))
    return {
        "nq_host": lambda: L.tsb_nq_search_ckpt(20, 12, 1, m_, M_, D, p, 0.0, C.byref(st)),
        "nq_host24": lambda: L.tsb_nq_search_ckpt(24, 12, 1, m_, M_, D, p, 0.0, C.byref(st)),
        "nq_device": lambda: L.tsb_nq_search_device_ckpt(20, 12, 1, m_, M_, D, p, 0.0, C.byref(st)),
        "pf_host": lambda: L.tsb_pfsp_search_ckpt(14, 1, 0, m_, M_, D, p, 0.0, C.byref(st)),
        "pf_host50": lambda: L.tsb_pfsp_search_ckpt_wide(50, 31, 1, 0, m_, M_, D, p, 0.0, C.byref(st)),
        "pf_device": lambda: L.tsb_pfsp_search_device_ckpt(14, 1, 0, m_, M_, D, 1, p, 0.0, C.byref(st)),
        "pf_device50": lambda: L.tsb_pfsp_search_device_ckpt_wide(50, 31, 1, 0, m_, M_, D, 1, p, 0.0, C.byref(st)),
    }


# file -> the searches that must refuse it (every one but the search that wrote it)
REFUSED = {
    "host N-Queens to the device form and the other width": (nq_host(), ["nq_device", "nq_host24", "pf_host"]),
    "device N-Queens to the host form": (nq_device(), ["nq_host", "nq_host24"]),
    "wide host N-Queens to the narrow host form": (nq_host(rec=25), ["nq_host", "nq_device"]),
    "host PFSP to the device forms": (pf_host(), ["pf_device", "pf_host50", "pf_device50", "nq_host"]),
    "device PFSP to the host forms": (pf_device(), ["pf_host", "pf_host50"]),
    "device PFSP, 2 pools, to the host form": (pf_device(pools=2, tasks=[(False, 0, [3, 1])]), ["pf_host"]),
    "host 50-job PFSP to the device and 20-job forms": (pf_host(rec=208, inst=31), ["pf_device50", "pf_host"]),
    "device 50-job PFSP to the host form": (pf_device(rec=208, inst=31), ["pf_host50"]),
    "host 20-job PFSP to the 50-job form": (pf_host(rec=88, inst=31), ["pf_host50"]),
}


@pytest.mark.parametrize("case", sorted(REFUSED))
def test_checkpoint_of_another_search_is_refused(L, tmp_path, case):
    content, refusers = REFUSED[case]
    path = tmp_path / "ck"
    path.write_bytes(content)
    for name in refusers:
        assert calls(L, path)[name]() == _lib.EINVAL, name
        assert path.read_bytes() == content and os.listdir(tmp_path) == ["ck"]


@pytest.mark.parametrize("states", [[], [3, 3], [0, 0], [1, 2, 3]])
@pytest.mark.parametrize("which", ["nq_host", "pf_host", "pf_host50"])
def test_host_task_without_exactly_one_pool_is_refused(L, tmp_path, which, states):
    """an unfinished host task with 0 or several pool states, or a finished one with any, is a damaged file"""
    make = {"nq_host": nq_host, "pf_host": pf_host, "pf_host50": lambda tasks: pf_host(rec=208, inst=31, tasks=tasks)}
    path = tmp_path / "ck"
    for tasks, D in (([(False, 0, states)], 1), ([(False, 0, [2]), (False, 1, states)], 2),
                     ([(True, 2, [2] if not states else states)], 1)):
        content = make[which](tasks=tasks)
        path.write_bytes(content)
        assert calls(L, path, D)[which]() == _lib.EINVAL
        assert path.read_bytes() == content and os.listdir(tmp_path) == ["ck"]


@pytest.mark.parametrize("which", ["nq_host", "nq_host24", "pf_host", "pf_host50"])
def test_host_checkpoint_is_taken(L, tmp_path, which):
    """well-formed host checkpoints (one pool per unfinished task, none for a finished one) pass the checks: without a
    device the search then fails as its twin does, and the file stays"""
    if L.tsb_device_count() > 0:
        pytest.skip("a CUDA device is present: the search would run")
    tasks = [(False, 0, [3]), (True, 2, []), (False, 0, [0])]
    content = {"nq_host": lambda: nq_host(tasks=tasks), "nq_host24": lambda: nq_host(rec=25, tasks=tasks),
               "pf_host": lambda: pf_host(tasks=tasks), "pf_host50": lambda: pf_host(rec=208, inst=31, tasks=tasks)}[which]()
    path = tmp_path / "ck"
    path.write_bytes(content)
    assert calls(L, path, D=3)[which]() == _lib.ENODEV
    assert path.read_bytes() == content

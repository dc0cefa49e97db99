"""The 50-job PFSP searches (tsb_pfsp_search_wide, tsb_pfsp_search_device_wide, tsb_pfsp_search_device_ckpt_wide)
where no GPU is needed: every argument is refused before any device call, and a checkpoint written for the other node
width is refused with TSB_EINVAL and left as it is."""
import ctypes as C
import os
import struct
import subprocess

import pytest

import tsb200
from tsb200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PFSP_DRIVER = os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200", "drivers", "pfsp_b200.out")


@pytest.fixture(scope="module")
def L():
    return tsb200.lib()


def calls(L, path, max_jobs=50, inst=31, lb=1, ub=1, m=25, M=1000, D=1, pools=1):
    st = _lib.SearchStats()
    p = os.fsencode(str(path))
    return (L.tsb_pfsp_search_wide(max_jobs, inst, lb, ub, m, M, D, C.byref(st)),
            L.tsb_pfsp_search_device_wide(max_jobs, inst, lb, ub, m, M, D, pools, C.byref(st)),
            L.tsb_pfsp_search_device_ckpt_wide(max_jobs, inst, lb, ub, m, M, D, pools, p, 0.0, C.byref(st)))


@pytest.mark.parametrize("args,code", [
    (dict(max_jobs=20), _lib.EINVAL), (dict(max_jobs=49), _lib.EINVAL), (dict(max_jobs=100), _lib.EINVAL),
    (dict(lb=3), _lib.EINVAL), (dict(lb=-1), _lib.EINVAL), (dict(ub=2), _lib.EINVAL), (dict(m=0), _lib.EINVAL),
    (dict(M=0), _lib.EINVAL), (dict(D=0), _lib.EINVAL), (dict(D=9), _lib.EINVAL),
    (dict(inst=30), _lib.EUNSUPPORTED), (dict(inst=61), _lib.EUNSUPPORTED), (dict(inst=1), _lib.EUNSUPPORTED),
    (dict(inst=0), _lib.EUNSUPPORTED), (dict(inst=121), _lib.EUNSUPPORTED),
    (dict(max_jobs=20, inst=30), _lib.EINVAL), (dict(inst=14, m=0), _lib.EINVAL)])
def test_arguments_refused_before_any_device_call(L, tmp_path, args, code):
    assert calls(L, tmp_path / "ck", **args) == (code, code, code)
    assert os.listdir(tmp_path) == []


@pytest.mark.parametrize("pools", [0, 5])
def test_pools_refused(L, tmp_path, pools):
    assert calls(L, tmp_path / "ck", pools=pools)[1:] == (_lib.EINVAL, _lib.EINVAL)


def test_declared_and_bound(L):
    for name in ("tsb_pfsp_search_wide", "tsb_pfsp_search_device_wide", "tsb_pfsp_search_device_ckpt_wide"):
        assert hasattr(L, name) and name in _lib.SYMBOLS
    assert callable(tsb200.pfsp_search_wide) and callable(tsb200.pfsp_search_device_wide)


def checkpoint(rec, inst, lb=1, ub=0, m=5, M=64, D=1, pools=1, nodes=3):
    """a well-formed one-task checkpoint (layout: csrc/search_ckpt.cpp) with `nodes` zero records of `rec` bytes"""
    b = b"TSB200CK" + struct.pack("<3I7i", 1, 2, rec, inst, lb, ub, m, M, D, pools)
    b += struct.pack("<QQqddQ", 0, 0, 2**63 - 1, 0.0, 0.0, 0)
    b += struct.pack("<5Qq2IQ", 0, 0, 0, 0, 0, 2**63 - 1, 0, 1, 0)
    b += struct.pack("<qQ", 2**63 - 1, nodes) + bytes(rec * nodes)
    h = 0xcbf29ce484222325
    for i in range(0, len(b) - len(b) % 8, 8):
        h = ((h ^ int.from_bytes(b[i:i + 8], "little")) * 0x100000001b3) & (2**64 - 1)
    for x in b[len(b) - len(b) % 8:]:
        h = ((h ^ x) * 0x100000001b3) & (2**64 - 1)
    return b + struct.pack("<Q", h ^ (h >> 29))


def test_checkpoint_of_the_other_width_is_refused(L, tmp_path):
    st = _lib.SearchStats()
    for rec, fn in ((88, "tsb_pfsp_search_device_ckpt_wide"), (208, "tsb_pfsp_search_device_ckpt")):
        path = tmp_path / f"ck{rec}"
        content = checkpoint(rec, 31)
        path.write_bytes(content)
        args = (31, 1, 0, 5, 64, 1, 1, os.fsencode(str(path)), 0.0, C.byref(st))
        rc = L.tsb_pfsp_search_device_ckpt_wide(50, *args) if rec == 88 else L.tsb_pfsp_search_device_ckpt(*args)
        assert rc == _lib.EINVAL, fn
        assert path.read_bytes() == content
    assert sorted(os.listdir(tmp_path)) == ["ck208", "ck88"]


def test_checkpoint_of_the_same_width_is_taken(L, tmp_path):
    """the same file with 208-byte records passes the checks: without a device the search then fails as its twin"""
    if L.tsb_device_count() > 0:
        pytest.skip("a CUDA device is present: the search would run")
    path = tmp_path / "ck"
    path.write_bytes(checkpoint(208, 31))
    st = _lib.SearchStats()
    assert L.tsb_pfsp_search_device_ckpt_wide(50, 31, 1, 0, 5, 64, 1, 1, os.fsencode(str(path)), 0.0,
                                              C.byref(st)) == _lib.ENODEV


def test_driver_max_jobs():
    r = subprocess.run([PFSP_DRIVER, "-h"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 1 and "--max-jobs" in r.stdout
    r = subprocess.run([PFSP_DRIVER, "--inst", "31", "--max-jobs", "30"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 2 and "--max-jobs" in r.stderr
    r = subprocess.run([PFSP_DRIVER, "--inst", "31", "--max-jobs", "50", "--devpool", "1"], capture_output=True,
                       text=True, timeout=60)
    assert "n = 50" in r.stdout

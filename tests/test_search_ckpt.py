"""The resumable device-pool searches (tsb_nq_search_device_ckpt, tsb_pfsp_search_device_ckpt) where no GPU is needed:
a checkpoint file that is damaged or is not one is refused with TSB_EINVAL before any device is touched, and the file
stays as it was; without a file and without a device the search fails as its twin does and writes nothing."""
import ctypes as C
import os
import subprocess

import pytest

import tsb200
from tsb200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVERS = os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200", "drivers")


@pytest.fixture(scope="module")
def L():
    return tsb200.lib()


def nq(L, path, N=12, M=1000, D=1, seconds=0.0, max_queens=20):
    st = _lib.SearchStats()
    return L.tsb_nq_search_device_ckpt(max_queens, N, 1, 25, M, D, os.fsencode(str(path)), seconds, C.byref(st))


def pfsp(L, path, inst=14, lb=1, ub=1, M=1000, D=1, pools=1, seconds=0.0):
    st = _lib.SearchStats()
    return L.tsb_pfsp_search_device_ckpt(inst, lb, ub, 25, M, D, pools, os.fsencode(str(path)), seconds, C.byref(st))


def test_new_symbols_and_code(L):
    for name in ("tsb_nq_search_device_ckpt", "tsb_pfsp_search_device_ckpt", "tsb_search_request_stop"):
        assert hasattr(L, name)
    assert _lib.ESTOPPED == -7 and L.tsb_strerror(-7)
    assert L.tsb_strerror(-7) != L.tsb_strerror(-100)
    e = tsb200.SearchStopped("where", _lib.SearchStats())
    assert isinstance(e, tsb200.TsbError) and e.code == _lib.ESTOPPED and e.stats.explored_tree == 0
    assert callable(tsb200.request_stop)


def test_missing_file_without_device(L, tmp_path):
    if L.tsb_device_count() > 0:
        pytest.skip("a CUDA device is present: the search would run")
    path = tmp_path / "ck"
    assert nq(L, path) == _lib.ENODEV
    assert pfsp(L, path) == _lib.ENODEV
    assert os.listdir(tmp_path) == []


@pytest.mark.parametrize("content", [b"", b"TSB2", b"TSB200CK", b"TSB200CK" + bytes(40), bytes(range(256)) * 3,
                                     b"XSB200CK" + bytes(200), b"\xff" * 4096])
def test_damaged_files_are_refused(L, tmp_path, content):
    """garbage, truncated files (the magic alone, a header cut short) and a wrong magic: TSB_EINVAL for both problems
    and every node width, the file's bytes unchanged and nothing else written"""
    path = tmp_path / "ck"
    path.write_bytes(content)
    assert nq(L, path) == _lib.EINVAL
    assert nq(L, path, N=22) == _lib.EINVAL
    assert nq(L, path, max_queens=24) == _lib.EINVAL
    assert pfsp(L, path) == _lib.EINVAL
    assert path.read_bytes() == content and os.listdir(tmp_path) == ["ck"]


def test_arguments(L, tmp_path):
    st = _lib.SearchStats()
    path = os.fsencode(str(tmp_path / "ck"))
    assert L.tsb_nq_search_device_ckpt(20, 12, 1, 25, 1000, 1, None, 0.0, C.byref(st)) == _lib.EINVAL
    assert L.tsb_nq_search_device_ckpt(20, 12, 1, 25, 1000, 1, b"", 0.0, C.byref(st)) == _lib.EINVAL
    assert L.tsb_nq_search_device_ckpt(20, 12, 1, 25, 1000, 1, path, float("nan"), C.byref(st)) == _lib.EINVAL
    assert L.tsb_nq_search_device_ckpt(21, 12, 1, 25, 1000, 1, path, 0.0, C.byref(st)) == _lib.EINVAL  # max_queens
    assert L.tsb_nq_search_device_ckpt(20, 12, 1, 25, 1000, 1, path, 0.0, None) == _lib.EINVAL
    assert nq(L, tmp_path / "ck", N=25) == _lib.EINVAL
    assert nq(L, tmp_path / "ck", D=9) == _lib.EINVAL
    assert pfsp(L, tmp_path / "ck", pools=5) == _lib.EINVAL
    assert pfsp(L, tmp_path / "ck", ub=2) == _lib.EINVAL
    assert os.listdir(tmp_path) == []


@pytest.mark.parametrize("name", ["nqueens_b200.out", "pfsp_b200.out"])
def test_driver_flags(name, tmp_path):
    exe = os.path.join(DRIVERS, name)
    r = subprocess.run([exe, "-h"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 1 and "--checkpoint" in r.stdout and "--time-limit" in r.stdout
    # a checkpoint needs the device pools, a time limit needs a checkpoint
    for args in (["--checkpoint", str(tmp_path / "ck")], ["--devpool", "1", "--time-limit", "5"]):
        r = subprocess.run([exe, *args], capture_output=True, text=True, timeout=60)
        assert r.returncode == 2 and r.stderr and "Size of the explored tree" not in r.stdout
    assert os.listdir(tmp_path) == []

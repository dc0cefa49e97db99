"""libtsb200_cbase.so without a device: what it exports, the record layouts it restates against the reference's own
headers, what the relinked reference drivers contain, the search goldens re-derived from the reference's sequential
program, and the refusals of evaluate_gpu that come before any CUDA call."""
import importlib.util
import json
import os
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200")
REF_OUT = os.path.join(ROOT, "oracle", "_ref")
SHIM = os.path.join(PKG, "libtsb200_cbase.so")


def _defined_dynamic(path):
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    return {line.split()[-1] for line in out.splitlines() if line.strip()}


def _ref_file(name):
    path = os.path.join(REF_OUT, name)
    if not os.path.exists(path):
        pytest.skip(f"oracle/_ref/{name} is built only where a checkout of the reference exists")
    return path


def test_shim_exports_only_evaluate_gpu_and_its_own_functions():
    assert _defined_dynamic(SHIM) == {"evaluate_gpu", "tsb_cbase_status", "tsb_cbase_release"}
    needed = subprocess.run(["readelf", "-d", SHIM], capture_output=True, text=True, check=True).stdout
    assert "[libtsb200.so]" in needed


def test_restated_layouts_equal_the_reference_headers():
    want = open(_ref_file("cbase_layout.txt")).read()
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "layout")
        subprocess.run(["gcc", "-O2", "-Wall", "-Werror", "-DTSB_CBASE", "-I", os.path.join(ROOT, "include"), "-o", exe,
                        os.path.join(ROOT, "oracle", "cbase_layout.c")], check=True)
        got = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
    assert got == want
    assert "Node sizeof 88\n" in got and "lb1_bound_data sizeof 32\n" in got and "lb2_bound_data sizeof 56\n" in got


@pytest.mark.parametrize("driver", ["pfsp_gpu_cuda", "pfsp_multigpu_cuda"])
def test_relinked_drivers_carry_no_kernel_of_the_reference(driver):
    orig, tsb = _ref_file(f"{driver}.out"), _ref_file(f"{driver}_tsb.out")
    syms = lambda p: subprocess.run(["nm", p], capture_output=True, text=True, check=True).stdout  # noqa: E731
    assert "evaluate_gpu_lb1" in syms(orig) and "evaluate_gpu_lb2" in syms(orig)
    t = syms(tsb)
    assert "evaluate_gpu_lb" not in t
    assert any(line.split() == ["U", "evaluate_gpu"] for line in t.splitlines())
    needed = subprocess.run(["readelf", "-d", tsb], capture_output=True, text=True, check=True).stdout
    assert "[libtsb200_cbase.so]" in needed


def _golden_script():
    spec = importlib.util.spec_from_file_location(
        "make_golden_cbase", os.path.join(ROOT, "tests", "golden", "make_golden_cbase.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("inst", [2, 7])
def test_goldens_rederive_from_the_reference_sequential_program(golden_dir, inst):
    exe = _ref_file("pfsp_c.out")
    gold = json.load(open(os.path.join(golden_dir, "pfsp_cbase_searches.json")))["searches"]
    mk = _golden_script()
    for name, lb in mk.LBS.items():
        assert mk.run(inst, lb, exe) == gold[f"ta{inst:03d}_{name}"], name


def test_golden_anchors(golden_dir):
    gold = json.load(open(os.path.join(golden_dir, "pfsp_cbase_searches.json")))["searches"]
    assert len(gold) == 21
    assert gold["ta014_lb1"] == {"tree": 2573652, "sol": 2648, "best": 1377}
    assert gold["ta014_lb2"] == {"tree": 144639, "sol": 0, "best": 1377}
    assert gold["ta003_lb1"] == {"tree": 2573133, "sol": 5689, "best": 1081}


# Runs in a child process, so that the sticky status starts at 0 and ends with the process.
_REFUSALS = r"""
import ctypes as C
from tsb200 import cbase
L = cbase.lib()
best = C.c_int(1377)
buf = (C.c_int * 64)()
p = C.cast(buf, C.POINTER(C.c_int))
def call(jobs, lb, size, nb_jobs=20, parents=True, bounds=True, best_p=C.pointer(best)):
    l1 = cbase.Lb1BoundData(p, p, p, nb_jobs, 5)
    L.evaluate_gpu(jobs, lb, size, 1, best_p, l1, cbase.Lb2BoundData(), C.addressof(buf) if parents else None,
                   C.addressof(buf) if bounds else None)
    return L.tsb_cbase_status()
codes = [L.tsb_cbase_status()]
codes.append(call(20, 1, 0))              # an empty chunk: nothing to do, no message
codes.append(call(50, 1, 50))             # jobs beyond the build's MAX_JOBS
codes.append(call(21, 1, 21))
L.tsb_cbase_release(); codes.append(L.tsb_cbase_status())
codes.append(call(20, 3, 20))             # unknown bound
L.tsb_cbase_release()
codes.append(call(20, -1, 20))
L.tsb_cbase_release()
codes.append(call(20, 1, -20))            # negative size
L.tsb_cbase_release()
codes.append(call(20, 1, 21))             # size not jobs * poolSize
L.tsb_cbase_release()
codes.append(call(20, 1, 20, nb_jobs=19)) # tables of another instance size
L.tsb_cbase_release()
codes.append(call(20, 1, 20, parents=False))
L.tsb_cbase_release()
codes.append(call(20, 0, 20, bounds=False))
L.tsb_cbase_release()
codes.append(call(20, 2, 20, best_p=None))  # lb2 reads *best
print(codes)
"""


def test_refusals_before_any_cuda_call():
    env = dict(os.environ, PYTHONPATH=PKG)
    r = subprocess.run([sys.executable, "-c", _REFUSALS], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0, r.stderr
    EINVAL, EUNSUPPORTED = -1, -6
    assert json.loads(r.stdout.strip()) == [0, 0, EUNSUPPORTED, EUNSUPPORTED, 0, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL,
                                            EINVAL, EINVAL, EINVAL]
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith("tsb200_cbase: evaluate_gpu(")]
    assert len(lines) == 10 and len(r.stderr.splitlines()) == 10, r.stderr
    assert "jobs=50" in lines[0] and "(-6)" in lines[0] and "(-6)" in lines[1]
    assert all("(-1)" in ln for ln in lines[2:]), lines

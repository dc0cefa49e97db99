"""The emulation drivers drivers/{nqueens,pfsp}_b200.out (the reference-compatible command line): exit codes of the
argument checks (no GPU needed: they return before any device is touched) and, on a GPU, their result lines against
the reference's counts (tests/golden/counts.json) and the oracle's (tests/golden/pfsp_searches.json)."""
import json
import os
import re
import subprocess

import pytest

import tsb200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVERS = os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200", "drivers")


def run(name, *args, timeout=600):
    exe = os.path.join(DRIVERS, name)
    assert os.path.exists(exe), f"{exe} is missing: build() makes it"
    return subprocess.run([exe, *map(str, args)], capture_output=True, text=True, timeout=timeout)


def field(text, pattern):
    m = re.search(pattern, text)
    assert m, (pattern, text)
    return m.group(1)


# ------------------------------------------------------------------------------------------ exit codes (CPU)
@pytest.mark.parametrize("name", ["nqueens_b200.out", "pfsp_b200.out"])
def test_help(name):
    r = run(name, "-h")
    assert r.returncode == 1 and "--m" in r.stdout


@pytest.mark.parametrize("args", [("--m", 0), ("--M", -3), ("--N", 0), ("--D", 0)])
def test_nq_bad_arguments(args):
    r = run("nqueens_b200.out", *args)
    assert r.returncode == 2 and r.stderr


@pytest.mark.parametrize("args", [("--m", 0), ("--inst", 121), ("--inst", 0), ("--lb", "lb3"), ("--ub", 2)])
def test_pfsp_bad_arguments(args):
    r = run("pfsp_b200.out", *args)
    assert r.returncode == 2 and r.stderr and "Size of the explored tree" not in r.stdout


@pytest.mark.parametrize("name,args,code", [("nqueens_b200.out", ("--D", 9), tsb200._lib.EINVAL),
                                            ("pfsp_b200.out", ("--D", 9), tsb200._lib.EINVAL),
                                            ("pfsp_b200.out", ("--inst", 31), None)])
def test_library_refusals(name, args, code):
    """the library's refusal (D > 8; a 50-job instance, which the search's 20-job nodes cannot hold) exits with 3
    and the library's own message"""
    r = run(name, *args)
    assert r.returncode == 3
    if code is not None:
        assert tsb200.lib().tsb_strerror(code).decode() in r.stderr
    else:
        assert re.search(r"tsb_pfsp_search: \S", r.stderr)
    assert "Size of the explored tree" not in r.stdout


# ------------------------------------------------------------------------------------------ result lines (GPU)
def counts(golden_dir):
    return json.load(open(os.path.join(golden_dir, "counts.json")))


def workload(text, D):
    shares = [float(x) for x in field(text, r"workload per GPU:([ \d.]+)\n").split()]
    assert len(shares) == D
    return shares


@pytest.mark.gpu
@pytest.mark.parametrize("devpool,D", [(0, 1), (1, 1), (0, 2), (1, 2)])
def test_nq_driver(devpool, D, golden_dir):
    r = run("nqueens_b200.out", "--N", 12, "--devpool", devpool, "--D", D)
    assert r.returncode == 0, r.stderr
    c = counts(golden_dir)["nqueens"]["12"]
    assert int(field(r.stdout, r"Size of the explored tree: (\d+)")) == c["tree"]
    assert int(field(r.stdout, r"Number of explored solutions: (\d+)")) == c["sol"]
    if D > 1:
        assert abs(sum(workload(r.stdout, D)) - 100.0) <= 0.05
    else:
        assert "workload per GPU" not in r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("devpool", [0, 1])
@pytest.mark.parametrize("lb,ub", [("lb1", 1), ("lb2", 1), ("lb2", 0)])
def test_pfsp_driver(lb, ub, devpool, golden_dir):
    r = run("pfsp_b200.out", "--inst", 14, "--lb", lb, "--ub", ub, "--devpool", devpool)
    assert r.returncode == 0, r.stderr
    if ub == 1:
        want = counts(golden_dir)["pfsp"][f"ta014_lb{tsb200.LB_NAMES[lb]}_ub1"]
    else:
        want = json.load(open(os.path.join(golden_dir, "pfsp_searches.json")))["searches"][f"ta014_{lb}_ub0_M50000_D1"]
    assert int(field(r.stdout, r"Size of the explored tree: (\d+)")) == want["tree"]
    assert int(field(r.stdout, r"Number of explored solutions: (\d+)")) == want["sol"]
    assert field(r.stdout, r"Optimal makespan: (.*)\n") == "1377" + (" (improved)" if ub == 0 else " (not improved)")


@pytest.mark.gpu
@pytest.mark.parametrize("devpool", [0, 1])
def test_pfsp_driver_workload(devpool, golden_dir):
    r = run("pfsp_b200.out", "--inst", 14, "--lb", "lb1", "--ub", 1, "--D", 3, "--M", 3000, "--devpool", devpool)
    assert r.returncode == 0, r.stderr
    want = counts(golden_dir)["pfsp"]["ta014_lb1_ub1"]
    assert int(field(r.stdout, r"Size of the explored tree: (\d+)")) == want["tree"]
    assert abs(sum(workload(r.stdout, 3)) - 100.0) <= 0.05

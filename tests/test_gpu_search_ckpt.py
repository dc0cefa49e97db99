"""The resumable device-pool searches on a GPU: a search chained through checkpoints (every invocation stops after one
library call per task, `seconds` = 0) ends with the stats of the uninterrupted search in every field but the times and
kernel_launches where the chunk sequence cannot depend on the stops (D = 1; PFSP with ub = 0), and with its tree, sol
and best where tasks steal; a stop requested from another thread; refusals of a real checkpoint that was damaged or is
given to another search; and the drivers' --checkpoint / --time-limit and SIGINT."""
import ctypes as C
import json
import os
import re
import signal
import subprocess
import threading
import time

import pytest

import tsb200
from tsb200 import _lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVERS = os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200", "drivers")
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "counts.json")))
EXACT = ("explored_tree", "explored_sol", "best", "offloads", "offloaded_parents", "steals")


@pytest.fixture(scope="module")
def L():
    return tsb200.lib()


def nq_call(L, path, N, M, D=1, max_queens=20, seconds=0.0):
    st = _lib.SearchStats()
    rc = L.tsb_nq_search_device_ckpt(max_queens, N, 1, 25, M, D, os.fsencode(str(path)), seconds, C.byref(st))
    return rc, st


def pfsp_call(L, path, inst, lb, ub, M, D=1, pools=1, seconds=0.0):
    st = _lib.SearchStats()
    rc = L.tsb_pfsp_search_device_ckpt(inst, lb, ub, 25, M, D, pools, os.fsencode(str(path)), seconds, C.byref(st))
    return rc, st


def chain(call, path):
    """rerun `call` until the search ends; (final stats, invocations); each stop leaves a checkpoint at `path`, the
    end removes it"""
    n = 0
    while True:
        rc, st = call()
        n += 1
        if rc != _lib.ESTOPPED:
            assert rc == _lib.OK, tsb200.lib().tsb_strerror(rc)
            assert not os.path.exists(path) and not os.path.exists(f"{path}.tmp")
            return st, n
        assert os.path.getsize(path) > 0
        assert n < 10000


def same(a, b, D):
    for f in EXACT:
        assert getattr(a, f) == getattr(b, f), f
    assert list(a.per_gpu_tree)[:D] == list(b.per_gpu_tree)[:D]
    assert a.t_step2 > 0 and a.kernel_launches > 0


# ------------------------------------------------------------------------------------------ N-Queens
@pytest.mark.parametrize("N,M", [(13, 256), (14, 512), (15, 2048)])
def test_nq_narrow_chain_is_the_uninterrupted_search(L, tmp_path, N, M):
    path = tmp_path / "nq.ck"
    got, n = chain(lambda: nq_call(L, path, N, M), path)
    want = tsb200.nqueens_search_device(N, 1, 25, M, 1)
    assert n >= 3
    same(got, want, 1)
    assert (got.explored_tree, got.explored_sol) == (GOLDEN["nqueens"][str(N)]["tree"], GOLDEN["nqueens"][str(N)]["sol"])


@pytest.mark.parametrize("N,M", [(12, 64), (13, 256), (14, 1024)])
def test_nq_wide_chain_is_the_uninterrupted_search(L, tmp_path, N, M):
    path = tmp_path / "nq24.ck"
    got, n = chain(lambda: nq_call(L, path, N, M, max_queens=24), path)
    want = tsb200.nqueens_search_device(N, 1, 25, M, 1, max_queens=24)
    assert n >= 3
    same(got, want, 1)
    assert (got.explored_tree, got.explored_sol) == (GOLDEN["nqueens"][str(N)]["tree"], GOLDEN["nqueens"][str(N)]["sol"])


def test_nq_two_tasks_with_stealing(L, tmp_path):
    """D = 2 on one GPU (the tasks wrap): the tasks steal, so only the totals are the search's"""
    path = tmp_path / "nq2.ck"
    got, n = chain(lambda: nq_call(L, path, 13, 256, D=2), path)
    assert n >= 2
    assert (got.explored_tree, got.explored_sol) == (GOLDEN["nqueens"]["13"]["tree"], GOLDEN["nqueens"]["13"]["sol"])
    assert sum(got.per_gpu_tree[:2]) > 0


def test_python_interface(tmp_path):
    path = tmp_path / "py.ck"
    stops = 0
    while True:
        try:
            st = tsb200.nqueens_search_device(12, 1, 25, 64, 1, max_queens=24, checkpoint=path, time_limit=0)
            break
        except tsb200.SearchStopped as e:
            stops += 1
            assert e.code == _lib.ESTOPPED and 0 < e.stats.explored_tree < GOLDEN["nqueens"]["12"]["tree"]
            assert path.exists()
    assert stops >= 2 and not path.exists()
    assert (st.explored_tree, st.explored_sol) == (GOLDEN["nqueens"]["12"]["tree"], GOLDEN["nqueens"]["12"]["sol"])
    # without a time limit it runs to the end in one call
    st = tsb200.pfsp_search_device(14, "lb1", 1, 25, 50000, checkpoint=path)
    assert (st.explored_tree, st.explored_sol, st.best) == (2573652, 2648, 1377) and not path.exists()


# ------------------------------------------------------------------------------------------ PFSP
@pytest.mark.parametrize("M", [50000, 500])
@pytest.mark.parametrize("pools", [1, 2])
def test_pfsp_ta014_lb1(L, tmp_path, pools, M):
    path = tmp_path / "pf.ck"
    got, n = chain(lambda: pfsp_call(L, path, 14, 1, 1, M, pools=pools), path)
    want = tsb200.pfsp_search_device(14, "lb1", 1, 25, M, 1, pools=pools)
    if M == 500:
        assert n >= 3
    same(got, want, 1)
    g = GOLDEN["pfsp"]["ta014_lb1_ub1"]
    assert (got.explored_tree, got.explored_sol, got.best) == (g["tree"], g["sol"], g["best"])


@pytest.mark.parametrize("M", [3000, 100])
@pytest.mark.parametrize("D", [1, 2])
def test_pfsp_ta002_lb2_ub0(L, tmp_path, D, M):
    """ub = 0: nothing moves between pools or tasks, so every field is the uninterrupted search's for any D"""
    path = tmp_path / "pf2.ck"
    got, n = chain(lambda: pfsp_call(L, path, 2, 2, 0, M, D=D, pools=2), path)
    want = tsb200.pfsp_search_device(2, "lb2", 0, 25, M, D, pools=2)
    if M == 100:
        assert n >= 2
    same(got, want, D)
    assert got.best == 1359


# ------------------------------------------------------------------------------------------ stop request
def test_stop_request_from_another_thread(L, tmp_path):
    path = tmp_path / "n17.ck"
    tsb200.nqueens_search_device(17, 1, 25, 50000, 1)  # (the device pools are cached: the next search starts warm)
    asked = []

    def ask():
        time.sleep(0.05)
        asked.append(time.perf_counter())
        tsb200.request_stop()

    th = threading.Thread(target=ask)
    th.start()
    rc, st = nq_call(L, path, 17, 50000, seconds=-1)
    back = time.perf_counter()
    th.join()
    assert rc == _lib.ESTOPPED and path.exists()
    latency = back - asked[0]
    print(f"\nN = 17 stop request to return: {latency * 1e3:.1f} ms; checkpoint {os.path.getsize(path)} bytes")
    assert 0 <= latency < 10
    assert 0 < st.explored_tree < GOLDEN["nqueens"]["17"]["tree"]
    rc, st = nq_call(L, path, 17, 50000, seconds=-1)  # (the request was cleared by the search that stopped on it)
    assert rc == _lib.OK and not path.exists()
    assert (st.explored_tree, st.explored_sol) == (GOLDEN["nqueens"]["17"]["tree"], GOLDEN["nqueens"]["17"]["sol"])


# ------------------------------------------------------------------------------------------ refusals
def test_refusals_of_a_real_checkpoint(L, tmp_path):
    nqp, pfp = tmp_path / "nq.ck", tmp_path / "pf.ck"
    assert nq_call(L, nqp, 13, 256)[0] == _lib.ESTOPPED
    assert pfsp_call(L, pfp, 14, 1, 1, 500, pools=2)[0] == _lib.ESTOPPED
    good_nq = nqp.read_bytes()

    def refused(path, call, data=None):
        if data is not None:
            path.write_bytes(data)
        before = path.read_bytes()
        assert call()[0] == _lib.EINVAL
        assert path.read_bytes() == before and not os.path.exists(f"{path}.tmp")

    flipped = bytearray(good_nq)
    flipped[len(flipped) // 2] ^= 0x10
    refused(nqp, lambda: nq_call(L, nqp, 13, 256), bytes(flipped))
    refused(nqp, lambda: nq_call(L, nqp, 13, 256), good_nq[: len(good_nq) // 2])
    refused(nqp, lambda: nq_call(L, nqp, 13, 256), good_nq[:-1])
    nqp.write_bytes(good_nq)
    refused(nqp, lambda: nq_call(L, nqp, 13, 512))                  # M
    refused(nqp, lambda: nq_call(L, nqp, 13, 256, D=2))             # D
    refused(nqp, lambda: nq_call(L, nqp, 14, 256))                  # N
    refused(nqp, lambda: nq_call(L, nqp, 13, 256, max_queens=24))   # node width
    refused(nqp, lambda: pfsp_call(L, nqp, 14, 1, 1, 256))          # problem
    refused(pfp, lambda: pfsp_call(L, pfp, 14, 1, 1, 500, pools=1))  # pools
    refused(pfp, lambda: pfsp_call(L, pfp, 14, 1, 0, 500, pools=2))  # ub
    refused(pfp, lambda: pfsp_call(L, pfp, 14, 2, 1, 500, pools=2))  # lb
    refused(pfp, lambda: nq_call(L, pfp, 13, 500))                  # a PFSP file to the N-Queens entry point
    # the untouched files still resume
    st, _ = chain(lambda: nq_call(L, nqp, 13, 256), nqp)
    assert (st.explored_tree, st.explored_sol) == (GOLDEN["nqueens"]["13"]["tree"], GOLDEN["nqueens"]["13"]["sol"])
    st, _ = chain(lambda: pfsp_call(L, pfp, 14, 1, 1, 500, pools=2), pfp)
    assert (st.explored_tree, st.explored_sol, st.best) == (2573652, 2648, 1377)


# ------------------------------------------------------------------------------------------ drivers
def run(name, *args, timeout=600):
    return subprocess.run([os.path.join(DRIVERS, name), *map(str, args)], capture_output=True, text=True,
                          timeout=timeout)


def result(text):
    return {k: re.search(p, text).group(1) for k, p in (("tree", r"Size of the explored tree: (\d+)"),
                                                         ("sol", r"Number of explored solutions: (\d+)"))}


@pytest.mark.parametrize("name,args", [("nqueens_b200.out", ("--N", 13, "--M", 256)),
                                       ("pfsp_b200.out", ("--inst", 14, "--lb", "lb1", "--M", 500))])
def test_driver_time_limit_chain(tmp_path, name, args):
    path = tmp_path / "drv.ck"
    whole = run(name, *args, "--devpool", 1)
    assert whole.returncode == 0, whole.stderr
    stops = 0
    while True:
        r = run(name, *args, "--devpool", 1, "--checkpoint", path, "--time-limit", 0)
        if r.returncode != 4:
            break
        stops += 1
        assert f"checkpoint written to {path}" in r.stdout and "Size of the explored tree" not in r.stdout
        assert stops < 100
    assert r.returncode == 0, r.stderr
    assert stops >= 2 and not path.exists()
    assert result(r.stdout) == result(whole.stdout)
    if name == "pfsp_b200.out":
        assert re.search(r"Optimal makespan: (.*)\n", r.stdout).group(1) == "1377 (not improved)"


def test_driver_sigint(tmp_path):
    """SIGINT to a running N = 17 search leaves a checkpoint; the same command finishes it (--M 2000: a few seconds
    of search, so that the signal lands inside it)"""
    path = tmp_path / "n17.ck"
    cmd = [os.path.join(DRIVERS, "nqueens_b200.out"), "--N", "17", "--M", "2000", "--devpool", "1",
           "--checkpoint", str(path)]
    p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    time.sleep(2.0)
    p.send_signal(signal.SIGINT)
    out, err = p.communicate(timeout=600)
    assert p.returncode == 4, (out, err)
    assert "rerun the same command to resume" in out and path.exists()
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert result(r.stdout) == {"tree": str(GOLDEN["nqueens"]["17"]["tree"]), "sol": str(GOLDEN["nqueens"]["17"]["sol"])}
    assert not path.exists()

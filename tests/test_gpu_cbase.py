"""libtsb200_cbase.so on the GPU: the reference's own C+CUDA PFSP drivers relinked against it (oracle/cbase.mk) find the
counts of the reference's sequential program (tests/golden/pfsp_cbase_searches.json) and of their unmodified builds,
and evaluate_gpu called in process through tsb200.cbase gives the oracle's bounds on the C baseline's tables, for
any chunk size, from several host threads, on the legacy default stream.  Every test ends with no message of the
library on stderr and tsb_cbase_status() == 0."""
import ctypes as C
import json
import os
import re
import subprocess
import tempfile
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_OUT = os.path.join(ROOT, "oracle", "_ref")
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "pfsp_cbase_searches.json")))["searches"]
LBS = {"lb1_d": 0, "lb1": 1, "lb2": 2}
INT_MAX = 2**31 - 1


def _exe(name):
    path = os.path.join(REF_OUT, name)
    if not os.path.exists(path):
        pytest.skip(f"oracle/_ref/{name} is built only where a checkout of the reference exists")
    return path


def _run(exe, *args):
    """the counts of the driver's final report; its stderr must hold no message of the library"""
    with tempfile.TemporaryDirectory() as cwd:  # (the drivers append to a stats file in their working directory)
        r = subprocess.run([exe, *map(str, args)], capture_output=True, text=True, cwd=cwd, timeout=600)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])
    assert "tsb200_cbase" not in r.stderr and "GPUassert" not in r.stderr, r.stderr
    g = lambda pat: int(re.findall(pat, r.stdout)[-1])  # noqa: E731
    return {"tree": g(r"Size of the explored tree: (\d+)"), "sol": g(r"Number of explored solutions: (\d+)"),
            "best": g(r"Optimal makespan: (\d+)")}


def _search_args(key):
    inst, lb = key.split("_", 1)
    return ["--inst", int(inst[2:]), "--lb", LBS[lb], "--ub", 1]


@pytest.mark.parametrize("m,M", [(25, 50000), (5, 1000)])
@pytest.mark.parametrize("key", sorted(GOLD))
def test_relinked_single_gpu_driver_matches_goldens(key, m, M):
    assert _run(_exe("pfsp_gpu_cuda_tsb.out"), *_search_args(key), "--m", m, "--M", M) == GOLD[key]


def test_relinked_single_gpu_driver_matches_its_original_under_ub0():
    """ta002 lb2 from an infinite incumbent: the chunk sequence follows the bounds, so any difference shows"""
    args = ["--inst", 2, "--lb", 2, "--ub", 0]
    want = _run(_exe("pfsp_gpu_cuda.out"), *args)
    assert _run(_exe("pfsp_gpu_cuda_tsb.out"), *args) == want
    assert want["best"] == 1359


def _gpus():
    import torch

    return torch.cuda.device_count()


@pytest.mark.parametrize("key", sorted(GOLD))
def test_relinked_multigpu_driver_matches_goldens(key):
    exe = _exe("pfsp_multigpu_cuda_tsb.out")
    for D in range(1, _gpus() + 1):
        assert _run(exe, *_search_args(key), "--D", D) == GOLD[key], D


def test_relinked_multigpu_driver_matches_its_original():
    args = ["--inst", 2, "--lb", 2, "--ub", 0, "--D", 1, "--perc", 25]
    want = _run(_exe("pfsp_multigpu_cuda.out"), *args)
    assert _run(_exe("pfsp_multigpu_cuda_tsb.out"), *args) == want


# ---------------------------------------------------------------- in process, through tsb200.cbase


@pytest.fixture
def cb(capfd):
    """tsb200.cbase with an empty cache; afterwards the status is 0 and stderr holds no message of the library"""
    from tsb200 import cbase

    cbase.release()
    yield cbase
    err = capfd.readouterr().err
    assert "tsb200_cbase" not in err, err
    assert cbase.status() == 0
    cbase.release()


def _parents(rng, n, jobs=20):
    from oracle import pyoracle as po

    nodes = np.zeros(n, dtype=po.PFSP_NODE_DTYPE)
    depth = rng.integers(1, jobs, size=n)
    nodes["depth"], nodes["limit1"] = depth, depth - 1
    nodes["prmu"][:, :jobs] = np.argsort(rng.random((n, jobs)), axis=1).astype(np.int32)
    return nodes


def _device(nodes):
    import torch

    return torch.from_numpy(nodes.view(np.uint8).copy()).cuda()


def _check(cb, tables, t, lb, nodes, best):
    """evaluate_gpu on `nodes` against the oracle on its live slots"""
    import torch
    from oracle import pyoracle as po

    n = len(nodes)
    bounds = torch.full((n * 20,), -7, dtype=torch.int32, device="cuda")
    cb.evaluate_gpu(20, lb, 20 * n, best, tables, _device(nodes), bounds)
    got = bounds.cpu().numpy().reshape(n, 20)
    want = po.pfsp_evaluate(t, lb, nodes, best).reshape(n, 20)
    live = po.pfsp_live_mask(nodes, 20)
    assert (got[live] == want[live]).all(), (lb, n, best)


@pytest.mark.parametrize("inst", [1, 14, 21])  # 5, 10 and 20 machines
def test_bounds_match_the_oracle_on_c_baseline_tables(cb, inst):
    from oracle import pyoracle as po

    t = po.tables(inst, heads_mode=1)
    tables = cb.upload_tables(t, "cuda:0")
    nodes = _parents(np.random.default_rng(inst), 3000)
    for lb in (0, 1, 2):
        _check(cb, tables, t, lb, nodes, INT_MAX)


def test_chunk_sizes_and_growth_past_the_first_call(cb):
    """the handle is built for the first call's chunk (1 parent); larger chunks go through the same handle"""
    from oracle import pyoracle as po

    t = po.tables(14, heads_mode=1)
    tables = cb.upload_tables(t, "cuda:0")
    rng = np.random.default_rng(5)
    for n in (1, 511, 512, 513, 20000, 3):
        for lb in (0, 1, 2):
            _check(cb, tables, t, lb, _parents(rng, n), INT_MAX)


def test_lb2_with_a_finite_incumbent(cb):
    from oracle import pyoracle as po

    t = po.tables(14, heads_mode=1)
    tables = cb.upload_tables(t, "cuda:0")
    nodes = _parents(np.random.default_rng(7), 4000)
    for best in (1377, 1300, 1000, 1):
        _check(cb, tables, t, 2, nodes, best)


def test_a_plain_cudaMemcpy_after_the_call_sees_the_bounds(cb):
    """the drivers' pattern: evaluate_gpu, then cudaMemcpy of the bounds with no synchronisation in between"""
    import torch
    from oracle import pyoracle as po

    rt = C.CDLL("libcudart.so.12")
    rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    t = po.tables(21, heads_mode=1)
    tables = cb.upload_tables(t, "cuda:0")
    n = 50000
    nodes = _parents(np.random.default_rng(11), n)
    parents_d = _device(nodes)
    want = {lb: po.pfsp_evaluate(t, lb, nodes, INT_MAX).reshape(n, 20) for lb in (0, 1, 2)}
    live = po.pfsp_live_mask(nodes, 20)
    for lb in (2, 0, 1, 2):
        bounds = torch.full((n * 20,), -7, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        host = np.zeros(n * 20, dtype=np.int32)
        cb.evaluate_gpu(20, lb, 20 * n, INT_MAX, tables, parents_d, bounds)
        assert rt.cudaMemcpy(host.ctypes.data, bounds.data_ptr(), host.nbytes, 2) == 0  # cudaMemcpyDeviceToHost
        assert (host.reshape(n, 20)[live] == want[lb][live]).all(), lb


def test_two_threads_with_their_own_tables_at_once(cb):
    from oracle import pyoracle as po

    work = {14: po.tables(14, heads_mode=1), 21: po.tables(21, heads_mode=1)}
    tables = {inst: cb.upload_tables(t, "cuda:0") for inst, t in work.items()}
    errors = []
    start = threading.Barrier(2)

    def task(inst):
        try:
            rng = np.random.default_rng(inst)
            start.wait()
            for i in range(12):
                _check(cb, tables[inst], work[inst], i % 3, _parents(rng, 500 + 700 * i), INT_MAX)
        except Exception as e:  # noqa: BLE001
            errors.append((inst, e))

    threads = [threading.Thread(target=task, args=(inst,)) for inst in work]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors


def test_new_table_pointers_get_a_new_handle(cb):
    """ta021 and ta025 have the same shape (20 x 20): only the table pointers tell their handles apart"""
    from oracle import pyoracle as po

    a, b = po.tables(21, heads_mode=1), po.tables(25, heads_mode=1)
    ta, tb = cb.upload_tables(a, "cuda:0"), cb.upload_tables(b, "cuda:0")
    nodes = _parents(np.random.default_rng(3), 2000)
    for lb in (0, 1, 2):
        _check(cb, ta, a, lb, nodes, INT_MAX)
        _check(cb, tb, b, lb, nodes, INT_MAX)
        assert (po.pfsp_evaluate(a, lb, nodes, INT_MAX) != po.pfsp_evaluate(b, lb, nodes, INT_MAX)).any()


def test_release_drops_the_handles(cb):
    """after a release the same pointers serve new tables (the documented way to change tables in place)"""
    import torch
    from oracle import pyoracle as po

    a, b = po.tables(21, heads_mode=1), po.tables(25, heads_mode=1)
    tables = cb.upload_tables(a, "cuda:0")
    nodes = _parents(np.random.default_rng(9), 1000)
    _check(cb, tables, a, 1, nodes, INT_MAX)
    cb.release()
    assert cb.status() == 0
    fresh = cb.upload_tables(b, "cpu")
    for k, v in tables.tensors.items():
        v.copy_(fresh.tensors[k])
    torch.cuda.synchronize()
    for lb in (0, 1, 2):
        _check(cb, tables, b, lb, nodes, INT_MAX)

"""CPU check of the route of 50-job device pools (csrc/pfr_tiers.h, pfw_takes, compiled as plain C++): which (M, K)
one launch of the persistent kernel of pfsp_wide_rounds.cuh takes.  It never takes a chunk beyond the K-pool capacity
of the 20-job kernel (the same 384-parent slice), takes only what the measured cutoffs allow (on an H100: one pool up
to 50 688, two up to 20 000, never three or four), and a launch that takes K pools takes any 2..K of them (the pools of
a shared launch leave it one by one)."""
import ctypes as C
import shutil
import subprocess

import pytest

from test_gpu_pfsp_pool_run_multi import pool_capacity
from test_ll_tag_window import CSRC

PROGRAM = r"""
#include "pfr_tiers.h"
extern "C" int takes(int sms, int pools, long long M) { return tsb::pfw_takes(sms, pools, M); }
extern "C" int max_m(int shared) { return shared ? tsb::PFW_MAX_M_SHARED : tsb::PFW_MAX_M_ONE; }
extern "C" int max_pools() { return tsb::PFW_MAX_POOLS_SHARED; }
"""


@pytest.fixture(scope="module")
def tiers(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("pfwtiers")
    src, so = d / "t.cpp", d / "t.so"
    src.write_text(PROGRAM)
    subprocess.run([cxx, "-std=c++17", "-O1", "-shared", "-fPIC", "-I", CSRC, "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    L.takes.argtypes = [C.c_int, C.c_int, C.c_longlong]
    return L


def test_h100_routes(tiers):
    assert [min(pool_capacity(132, K), tiers.max_m(K > 1)) for K in (1, 2)] == [50688, 20000]
    for K in (1, 2):
        edge = min(pool_capacity(132, K), tiers.max_m(K > 1))
        assert tiers.takes(132, K, edge) and not tiers.takes(132, K, edge + 1), K
        assert tiers.takes(132, K, 1)
    assert tiers.max_pools() == 2 and not tiers.takes(132, 3, 1) and not tiers.takes(132, 4, 1)


def test_every_sm_count(tiers):
    Ms = sorted({1, 64, 1000, 6000, 20000, 25344, 33792, 50000, 50688, 50689, 100000} |
                {tiers.max_m(0), tiers.max_m(0) + 1, tiers.max_m(1), tiers.max_m(1) + 1})
    for sms in range(1, 300):
        for M in Ms:
            got = [bool(tiers.takes(sms, K, M)) for K in (1, 2, 3, 4)]
            for K in (1, 2, 3, 4):
                assert got[K - 1] == (K <= tiers.max_pools() and M <= pool_capacity(sms, K) and
                                      M <= tiers.max_m(K > 1)), (sms, M, K)
            for K in (3, 4):  # K pools taken -> any 2..K taken
                assert not got[K - 1] or all(got[1:K - 1]), (sms, M, K)
    assert not tiers.takes(132, 0, 1) and not tiers.takes(132, 5, 1)

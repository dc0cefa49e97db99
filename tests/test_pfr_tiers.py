"""CPU check of the capacities of the persistent PFSP kernel per pool (csrc/pfr_tiers.h), compiled as plain C++:
the header agrees with the formulas the GPU tests size their chunks by, on every SM count, and gives the H100's
table (132 SMs: 50 688 parents per pool for one or two pools, 33 792 for three, 25 344 for four)."""
import ctypes as C
import shutil
import subprocess

import pytest

from test_gpu_pfsp_pool_run_multi import ctas_per_pool, pool_capacity
from test_ll_tag_window import CSRC

PROGRAM = r"""
#include "pfr_tiers.h"
static_assert(tsb::pf_pool_capacity(132, 2) == 50688, "H100, two pools");
extern "C" int ctas(int sms, int pools) { return tsb::pf_ctas_per_pool(sms, pools); }
extern "C" long long capacity(int sms, int pools) { return tsb::pf_pool_capacity(sms, pools); }
"""


@pytest.fixture(scope="module")
def tiers(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("pfrtiers")
    src, so = d / "t.cpp", d / "t.so"
    src.write_text(PROGRAM)
    subprocess.run([cxx, "-std=c++17", "-O1", "-shared", "-fPIC", "-I", CSRC, "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    L.capacity.restype = C.c_longlong
    return L


def test_h100_table(tiers):
    assert [tiers.ctas(132, K) for K in (1, 2, 3, 4)] == [132, 132, 88, 66]
    assert [tiers.capacity(132, K) for K in (1, 2, 3, 4)] == [50688, 50688, 33792, 25344]


def test_every_sm_count(tiers):
    for sms in range(1, 300):
        for K in (1, 2, 3, 4):
            assert tiers.ctas(sms, K) == ctas_per_pool(sms, K), (sms, K)
            assert tiers.capacity(sms, K) == pool_capacity(sms, K), (sms, K)
            assert K * tiers.ctas(sms, K) <= (1 if K == 1 else 2) * sms  # one CTA per SM, or two

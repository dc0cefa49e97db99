"""CPU check of csrc/xfer_route.h, compiled as plain C++: the route rule of tsb_*_evaluate (what tsb_*_last_xfer
reports), and the small N-Queens kernel's loads at the end of a chunk, for arrays that end at a page boundary — the case
no GPU test may place in a registered range."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from test_ll_tag_window import CSRC, ROOT

PAGE = 4096
AUTO, MEMCPY, ZEROCOPY = 0, 1, 2
R_ZC, R_PIPE, R_IN, R_OUT = 1, 2, 4, 8
BASE = 1 << 30

PROGRAM = r"""
#include "xfer_route.h"
static_assert(tsb::xfer_route(TSB_XFER_AUTO, true, true, 0, 16, true, 50000, 131072, 262144) == TSB_XFER_ROUTE_ZEROCOPY, "");
extern "C" int route(int mode, int in_locked, int out_locked, uintptr_t in, uintptr_t out, int can_map, long long count,
                     long long pipe_min, long long pipe_chunk) {
  return tsb::xfer_route(mode, in_locked, out_locked, in, out, can_map, count, pipe_min, pipe_chunk);
}
extern "C" int small_words(int np, int rec) { return tsb::nq_small_words(np, rec); }
"""


@pytest.fixture(scope="module")
def xr(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("xferroute")
    src, so = d / "x.cpp", d / "x.so"
    src.write_text(PROGRAM)
    subprocess.run([cxx, "-std=c++17", "-O1", "-shared", "-fPIC", "-I", CSRC, "-I", os.path.join(ROOT, "include"),
                    "-o", str(so), str(src)], check=True)
    L = C.CDLL(str(so))
    L.route.argtypes = [C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_int, C.c_longlong, C.c_longlong,
                        C.c_longlong]
    return L


def test_route_rule(xr):
    for mode in (AUTO, MEMCPY, ZEROCOPY):
        for li in (0, 1):
            for lo in (0, 1):
                for a_in, a_out in ((0, 0), (8, 0), (0, 4), (16, 32)):
                    for can_map in (0, 1):
                        for count in (1, 1024, 1025, 131071, 131072, 262144, 262145):
                            zc = li and lo and a_in % 16 == 0 and a_out % 16 == 0 and can_map and mode != MEMCPY
                            want = R_ZC if zc else ((R_PIPE if count >= 131072 and count > 262144 else 0)
                                                    | (0 if li else R_IN) | (0 if lo else R_OUT))
                            got = xr.route(mode, li, lo, BASE + a_in, BASE + a_out, can_map, count, 131072, 262144)
                            assert got == want, (mode, li, lo, a_in, a_out, can_map, count)
    # the thresholds the GPU tests set (TSB200_PIPE_MIN=1, TSB200_PIPE_CHUNK=1024)
    assert xr.route(AUTO, 1, 1, BASE, BASE, 1, 1025, 1, 1024) == R_ZC
    assert xr.route(MEMCPY, 1, 1, BASE, BASE, 1, 1025, 1, 1024) == R_PIPE
    assert xr.route(MEMCPY, 1, 1, BASE, BASE, 1, 1024, 1, 1024) == 0
    assert xr.route(ZEROCOPY, 0, 1, BASE, BASE, 1, 1, 1, 1024) == R_IN  # a forced zero-copy that cannot: copies


def test_small_nq_kernel_reads_end_at_the_last_record(xr):
    """each CTA of the small N-Queens kernel (128 parents of 21 bytes) loads whole 16-byte words and then single
    bytes: its last read is its last record's last byte, so an aligned array that ends at a page boundary is never read
    past (the loads before this change rounded the last CTA up to whole words: up to 15 bytes into the next page)"""
    rec, cta = 21, 128
    rounded_up_past = 0
    for count in range(1, 4 * cta + 1):
        start = PAGE * 64 - count * rec  # the array ends at a page boundary
        covered, last = 0, start
        for p0 in range(0, count, cta):
            np_ = min(cta, count - p0)
            words = xr.small_words(np_, rec)
            assert 16 * words <= np_ * rec < 16 * words + 16, (count, p0)
            covered += np_ * rec  # words [0, words), then bytes [16 * words, np * rec): the CTA's records exactly
            last = start + p0 * rec + np_ * rec
            rounded_up_past += (np_ * rec + 15) // 16 * 16 > np_ * rec
        assert covered == count * rec and last == PAGE * 64
    assert rounded_up_past > 0

"""CPU check of the host's clear decision for the 16-bit node tags of the persistent N-Queens kernel
(tsb::ll_tag_window, csrc/ll_tiers.h), compiled as plain C++: over long sequences of launches of any length, every
launch can run at least one round, never uses an epoch more than LL_TAG_SPAN past the last clear (so no stale tag
can alias a live one, nq_rounds_ll.cuh), and clears at most once per LL_TAG_SPAN / 2 epochs."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gpu-accelerated-tree-search-chapel_b200", "csrc")
SPAN = 65535

PROGRAM = r"""
#include "ll_tiers.h"
static_assert(tsb::LL_TAG_SPAN == 65535u, "tags 1 .. 65535");
extern "C" unsigned tag_window(unsigned epoch, unsigned clear_epoch, long long max_rounds, int* clear) {
  const tsb::LlTagWindow w = tsb::ll_tag_window(epoch, clear_epoch, max_rounds);
  *clear = w.clear ? 1 : 0;
  return w.epoch_last;
}
"""


@pytest.fixture(scope="module")
def window(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("tagwin")
    src, so = d / "w.cpp", d / "w.so"
    src.write_text(PROGRAM)
    subprocess.run([cxx, "-std=c++17", "-O1", "-shared", "-fPIC", "-I", CSRC, "-o", str(so), str(src)], check=True)
    fn = C.CDLL(str(so)).tag_window
    fn.restype = C.c_uint
    fn.argtypes = [C.c_uint, C.c_uint, C.c_longlong, C.POINTER(C.c_int)]

    def call(epoch, clear_epoch, max_rounds):
        c = C.c_int()
        last = fn(epoch, clear_epoch, max_rounds, C.byref(c))
        return c.value == 1, last
    return call


def test_window_edges(window):
    got = [window(*q) for q in [
        (0, 0, 10 ** 9),          # fresh arena: the whole window
        (0, 0, 1),
        (SPAN - 1, 0, 1),         # one epoch left: enough for one round
        (SPAN - 1, 0, 2),         # ... not for two: clear
        (SPAN, 0, 1),             # none left: clear
        (SPAN // 2 + 1, 0, 10 ** 9),  # exactly LL_TAG_SPAN / 2 left: no clear
        (SPAN // 2 + 2, 0, 10 ** 9),  # one fewer: clear
        (100, 50, 0),
    ]]
    assert got == [(False, SPAN), (False, SPAN), (False, SPAN), (True, 2 * SPAN - 1), (True, 2 * SPAN),
                   (False, SPAN), (True, SPAN // 2 + 2 + SPAN), (False, 50 + SPAN)]


@pytest.mark.parametrize("seed", range(4))
def test_launch_sequences_keep_the_window(window, seed):
    """random launches (round budgets from 1 to beyond the window, launches that stop early): the host's loop of
    rounds_run (NqRounds::prepare), one decision at a time"""
    rng = np.random.default_rng(seed)
    epoch, clear, clears = 0, 0, 0
    for _ in range(3000):
        budget = int(rng.choice([1, 2, 3, int(rng.integers(1, 5000)), int(rng.integers(1, 3 * SPAN)), 10 ** 12]))
        while budget > 0:
            c, last = window(epoch, clear, budget)
            if c:
                assert epoch - clear >= SPAN // 2
                clear = epoch
                clears += 1
            assert last > epoch and last - clear <= SPAN
            ran = min(budget, last - epoch)
            if rng.random() < 0.3:  # (the pool ran dry or left for room)
                ran = int(rng.integers(0, ran + 1))
                budget = 0
            epoch += ran
            budget -= ran
    assert clears > 10

// xfer_route.h — what the host-buffer entry points decide from plain addresses and counts, kept free of CUDA so that
// the tests compile it as plain C++ and check the cases no GPU test may run (arrays that end at a page boundary):
//   * xfer_route: the route of one tsb_*_evaluate call (TSB_XFER_ROUTE_* bits of tsb200.h);
//   * nq_small_words: the part of a CTA's parents the small N-Queens kernel loads as whole 16-byte words.
#pragma once
#include <cstdint>

#include "tsb200.h"

namespace tsb {

// Route of one host-buffer evaluate call of `count` records with the transfer mode `mode` (TSB_XFER_*).  Zero-copy
// needs both arrays registered, both 16-byte aligned and a device that can use registered host pointers; AUTO takes
// it whenever it can, a forced TSB_XFER_ZEROCOPY that cannot falls back to the copies.  Copies of unregistered arrays
// are staged through the handle's pinned buffers, and chunks of at least pipe_min and more than pipe_chunk records
// are split over two streams.
constexpr int xfer_route(int mode, bool in_locked, bool out_locked, uintptr_t in, uintptr_t out, bool can_map,
                         long long count, long long pipe_min, long long pipe_chunk) {
  const bool zc_ok = in_locked && out_locked && ((in | out) & 15) == 0 && can_map;
  if (zc_ok && mode != TSB_XFER_MEMCPY) return TSB_XFER_ROUTE_ZEROCOPY;
  return (count >= pipe_min && count > pipe_chunk ? TSB_XFER_ROUTE_PIPELINED : 0) |
         (in_locked ? 0 : TSB_XFER_ROUTE_IN_STAGED) | (out_locked ? 0 : TSB_XFER_ROUTE_OUT_STAGED);
}

// The small N-Queens kernel loads the `np` parents of a CTA (np * rec bytes from a 16-byte aligned start) as this many
// whole 16-byte words and the rest byte by byte: it never reads past the CTA's last record, which in zero-copy mode
// is the last record of the caller's registered host array (whose end may be the end of a mapped page).
#ifdef __CUDACC__
__host__ __device__
#endif
constexpr int nq_small_words(int np, int rec) { return np * rec / 16; }

}  // namespace tsb

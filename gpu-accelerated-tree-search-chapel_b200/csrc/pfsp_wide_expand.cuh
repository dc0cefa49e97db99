// pfsp_wide_expand.cuh — one evaluate + generate_children round on the device for 208-byte tsb_pfsp_node50 records
// (the reference built with MAX_JOBS = 50), the two-kernel shape of pfsp_expand.cuh:
//   pfsp_wide_expand_count : the bounds of pfsp_wide_kernel (pw_parent_bounds) on parents read in place from the
//                            arena's extents, in tiles of PW_TILE; epilogue: one 64-bit child mask per parent (slot
//                            k > limit1, not a leaf, lb < best), one child count per tile, leaf count and leaf minimum
//                            into ExpandState
//   pfsp_wide_expand_build : offsets of the CTA's own tiles (expand_own_offsets), then per tile: the children listed
//                            in the reference's order (parent, then slot) and stored as whole 16-byte words, coalesced
//                            (208 = 13 x 16: every child of the packed output is 16-byte aligned)
// A child is {depth + 1, limit1 + 1, prmu with prmu[depth] <=> prmu[k]} (pfsp_gpu_chpl.chpl:273-303).  `best` is the
// launch value for the whole round; the host redoes a round whose leaves lowered it (tsb200_api.cu, slow path).
#pragma once
#include "expand_common.cuh"
#include "pfsp_wide.cuh"

namespace tsb {

constexpr int PW_WORDS = PW_REC / 16;              // 13 16-byte words per record
constexpr int PW_EXP_ITEMS = PW_TILE * PW_MAXJ;    // children of one tile at most (a root has 50)
static_assert(PW_REC % 16 == 0 && PW_THREADS == 64, "two warps, one parent per thread, 16-byte records");

// the records [r0, r1) of linear tile `lin` (absolute tile `at`) into in[] at their tile positions
__device__ __forceinline__ void pw_load_tile(int32_t* in, const uint8_t* __restrict__ arena, long long at, int r0, int r1) {
  const uint4* src = reinterpret_cast<const uint4*>(arena + (at * PW_TILE + r0) * PW_REC);
  uint4* dst = reinterpret_cast<uint4*>(in + r0 * (PW_REC / 4));
  for (int i = threadIdx.x; i < (r1 - r0) * PW_WORDS; i += PW_THREADS) dst[i] = src[i];
}

struct PfspWideCountSmem {
  PfspWideSmem core;  // tables, the tile's parents and their bounds
  int red[2];
};

template <int KIND, int M>
__global__ void __launch_bounds__(PW_THREADS) pfsp_wide_expand_count_kernel(const uint8_t* __restrict__ arena,
                                                                           const __grid_constant__ ExpandParams prm,
                                                                           const PfspWideTables* __restrict__ tables,
                                                                           unsigned long long* __restrict__ cmask,
                                                                           int* __restrict__ tile_sums,
                                                                           ExpandState* __restrict__ st) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  PfspWideCountSmem& sm = *reinterpret_cast<PfspWideCountSmem*>(smem_raw);
  const int t = threadIdx.x;
  pw_stage_tables<KIND>(&sm.core.tab, tables);
  const PfspWideTables& tab = sm.core.tab;
  const int best = prm.best;
  unsigned my_solutions = 0;
  for (int lin = blockIdx.x; lin < prm.n_tiles; lin += gridDim.x) {
    long long at, lo, hi;
    piece_of(prm, lin, PW_TILE, at, lo, hi);
    const int r0 = static_cast<int>(lo - at * PW_TILE), r1 = static_cast<int>(hi - at * PW_TILE);
    pw_load_tile(sm.core.in, arena, at, r0, r1);
    __syncthreads();  // (also: the tables, on the first tile)
    const int jobs = tab.jobs;
    unsigned long long m = 0;
    int leaves = 0;
    if (t >= r0 && t < r1) {
      const int32_t* node = sm.core.in + t * (PW_REC / 4);
      int32_t* b = sm.core.out + t * jobs;
      pw_parent_bounds<KIND, M>(tab, node, sm.core.fc + t, best, b);
      const int limit1 = min(max(node[1], -1), jobs - 1);
      if (node[0] + 1 == jobs) {  // every child is a leaf (pfsp_gpu_chpl.chpl:283-288)
        int leaf_lb = 0x7FFFFFFF;
        for (int k = limit1 + 1; k < jobs; k++) leaf_lb = min(leaf_lb, b[k]);
        leaves = jobs - 1 - limit1;
        if (leaf_lb < best) atomicMin(&st->best, leaf_lb);
      } else {
        for (int k = limit1 + 1; k < jobs; k++)
          if (b[k] < best) m |= 1ull << k;
      }
    }
    cmask[static_cast<long long>(lin) * PW_TILE + t] = m;
    int packed = __popcll(m) | (leaves << 16);  // children and leaves of a tile <= 64 * 50 < 2^16
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) packed += __shfl_xor_sync(0xFFFFFFFFu, packed, o);
    if ((t & 31) == 0) sm.red[t >> 5] = packed;
    __syncthreads();
    if (t == 0) {
      const int tot = sm.red[0] + sm.red[1];
      tile_sums[lin] = tot & 0xFFFF;
      my_solutions += static_cast<unsigned>(tot >> 16);
    }
    __syncthreads();  // the next tile overwrites the parents and red[]
  }
  if (t == 0 && my_solutions) atomicAdd(&st->solutions, static_cast<unsigned long long>(my_solutions));
}

struct PfspWideBuildSmem {
  alignas(16) int32_t in[PW_TILE * (PW_REC / 4)];
  uint16_t item[PW_EXP_ITEMS];  // (record << 6) | slot, in child order
  int warp_tot[2];
  ScanSmem scan;
};

__global__ void __launch_bounds__(PW_THREADS) pfsp_wide_expand_build_kernel(const uint8_t* __restrict__ arena,
                                                                           const __grid_constant__ ExpandParams prm,
                                                                           const unsigned long long* __restrict__ cmask,
                                                                           const int* __restrict__ tile_sums,
                                                                           uint8_t* __restrict__ children,
                                                                           ExpandState* __restrict__ st,
                                                                           ExpandResult* __restrict__ res) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  PfspWideBuildSmem& sm = *reinterpret_cast<PfspWideBuildSmem*>(smem_raw);
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int first = blockIdx.x, stride = gridDim.x;
  expand_own_offsets<PW_THREADS>(sm.scan, tile_sums, prm.n_tiles, first, stride);
  expand_publish(sm.scan, st, res, prm.epoch, 1);  // st->best restarts at INT_MAX every round
  unsigned it = 0;
  for (int lin = first; lin < prm.n_tiles; lin += stride, it++) {
    const int total = sm.scan.cnt[it];
    if (total == 0) continue;  // (uniform across the CTA)
    long long at, lo, hi;
    piece_of(prm, lin, PW_TILE, at, lo, hi);
    const unsigned long long cm = cmask[static_cast<long long>(lin) * PW_TILE + t];  // 0 outside [lo, hi)
    const int mine = __popcll(cm);
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) sm.warp_tot[wid] = incl;
    pw_load_tile(sm.in, arena, at, static_cast<int>(lo - at * PW_TILE), static_cast<int>(hi - at * PW_TILE));
    __syncthreads();  // (A) warp totals, parents
    int pos = (wid ? sm.warp_tot[0] : 0) + incl - mine;  // this parent's first child within the tile
    for (unsigned long long m = cm; m; m &= m - 1) sm.item[pos++] = static_cast<uint16_t>((t << 6) | (__ffsll(m) - 1));
    __syncthreads();  // (B) items
    int4* g = reinterpret_cast<int4*>(children + static_cast<long long>(sm.scan.own[it]) * PW_REC);
    for (int i = t; i < total * PW_WORDS; i += PW_THREADS) {  // word w of child c: consecutive threads, consecutive words
      const int c = i / PW_WORDS, w = i - c * PW_WORDS;
      const int item = sm.item[c];
      const int32_t* src = sm.in + (item >> 6) * (PW_REC / 4);
      const int k = item & 63, depth = src[0];
      const int4 v = reinterpret_cast<const int4*>(src)[w];
      int e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; j++) {  // int 4w + j of the record: depth, limit1, prmu[0..50)
        const int x = 4 * w + j;
        if (x == 0) e[j] = depth + 1;
        else if (x == 1) e[j] = src[1] + 1;
        else if (x == 2 + depth) e[j] = src[2 + k];  // child.prmu[depth] <=> child.prmu[k]
        else if (x == 2 + k) e[j] = src[2 + depth];
      }
      g[i] = make_int4(e[0], e[1], e[2], e[3]);
    }
    __syncthreads();  // (C) the next tile overwrites parents, items and warp totals
  }
}

}  // namespace tsb

// nq_expand.cuh — N-Queens evaluation + child generation on the device (SURVEY §8f rows 1 and 3).
//
// Restates, on the GPU, evaluate_gpu (nqueens_gpu_chpl.chpl:97-123) followed by generate_children
// (:126-149): for every parent p of a chunk, in order, and every slot j = depth..N-1, in order, whose
// queen is safe, emit the child {depth+1, board with board[depth] <=> board[j]}; a parent with
// depth == N counts as one explored solution.  The children come out PACKED and IN THE REFERENCE'S
// ORDER, so a pool that appends them is byte-identical to the reference's pool after the same round.
//
// Three kernels per chunk (expand_common.cuh), the chunk read in place from the pool arena:
//   nq_expand_count : the evaluator of nq_kernel.cuh (TMA-pipelined tiles of 512 parents), but instead of N
//                     label bytes per parent it writes the tile's ITEMS — one uint16 (parent << 5 | slot) per
//                     child, in child order (block scan of the per-parent counts) — and one child count per
//                     tile; parents with depth == N are counted as solutions
//   nq_expand_build : tile counts -> offsets of the CTA's own tiles (prologue); per tile (2-stage TMA prefetch
//                     of parents + items, no scan left to do): children built in shared
//                     memory as a contiguous byte image at the 16-byte phase of their destination — one thread
//                     per child, the parent read as six aligned words, the two queens swapped by an XOR patch
//                     in registers, realigned by funnel shifts and stored as words (+ the few bytes of the two
//                     words it shares with its neighbours) — and written with one TMA bulk store plus < 16
//                     head / tail bytes (21-byte records land at any alignment)
// HBM traffic per parent: 21 B (count) + 2 B per child (items, written and re-read) and 21 B (mostly L2) + 21 B per
// child (build).  Every kernel is a template over the record width R (nq_kernel.cuh): 21 or 25 bytes; a 25-byte
// child is seven words instead of six, and the items stay (parent << 5 | slot) for slots up to 23.
#pragma once
#include "expand_common.cuh"
#include "nq_kernel.cuh"

namespace tsb {

#ifndef TSB_EXP_CAP
#define TSB_EXP_CAP 1024
#endif
constexpr int EXP_CAP = TSB_EXP_CAP;  // children per pass of the shared staging image (a tile averages ~512; denser tiles take several passes)

template <int N, int Q, int R>
__device__ __forceinline__ uint32_t nq_child_mask(NqParent<N, Q, R>& p) {
  const uint32_t S = ~p.U;
  uint32_t cm = 0;
#pragma unroll
  for (int k = 0; k < N; k++) {
    const uint32_t x = shf_r_wrap(S, 0u, p.amt[k]) & 1u;  // bit board[k] of the safe-value mask
    asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(cm) : "r"(x), "r"(1u << k));  // cm |= x << k on the FMA pipe
  }
  return cm & shl_clamp(0xFFFFFFFFu, p.depth);  // only slots k >= depth exist
}

// evaluate the four parents of this thread: child masks + number of leaves (depth == N)
template <int N, int R>
__device__ __forceinline__ void nq_eval_quad(const uint8_t* in_tile, long long pos0, long long lo, long long hi,
                                             uint32_t (&cm)[4], int& leaves) {
  const int t = threadIdx.x;
  const uint32_t* in_w = reinterpret_cast<const uint32_t*>(in_tile) + R * t;
  uint32_t w[R];
#pragma unroll
  for (int i = 0; i < R; i++) w[i] = in_w[i];
  NqParent<N, 0, R> p0;
  NqParent<N, 1, R> p1;
  NqParent<N, 2, R> p2;
  NqParent<N, 3, R> p3;
  p0.init(w);
  p1.init(w);
  p2.init(w);
  p3.init(w);
  const uint32_t dep[4] = {p0.depth, p1.depth, p2.depth, p3.depth};
  bool valid[4];
  uint32_t dmax = 0;
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const long long p = pos0 + 4 * t + q;
    valid[q] = p >= lo && p < hi;
    if (valid[q]) dmax = max(dmax, dep[q]);  // records outside the chunk hold arbitrary bytes
  }
  dmax = min(dmax, static_cast<uint32_t>(R - 1));
#pragma unroll
  for (int j = 0; j < (N + 3) / 4; j++) {
    if (dmax > 4u * j) {
      switch (j) {
#define TSB_ROWS(J)                          \
  case J:                                    \
    p0.template rows<4 * J, 4 * J + 4>();    \
    p1.template rows<4 * J, 4 * J + 4>();    \
    p2.template rows<4 * J, 4 * J + 4>();    \
    p3.template rows<4 * J, 4 * J + 4>();    \
    break;
        TSB_ROWS(0) TSB_ROWS(1) TSB_ROWS(2) TSB_ROWS(3) TSB_ROWS(4) TSB_ROWS(5)
#undef TSB_ROWS
      }
    }
  }
  cm[0] = nq_child_mask(p0);
  cm[1] = nq_child_mask(p1);
  cm[2] = nq_child_mask(p2);
  cm[3] = nq_child_mask(p3);
  leaves = 0;
#pragma unroll
  for (int q = 0; q < 4; q++) {
    if (!valid[q] || dep[q] >= static_cast<uint32_t>(N)) cm[q] = 0;
    if (valid[q] && dep[q] == static_cast<uint32_t>(N)) leaves++;
  }
}

// ------------------------------------------------------------------------------------------- count
template <int R>
struct NqCountSmem {
  alignas(128) uint8_t in[2][NQ_TILE * R];
  alignas(8) uint64_t full[2];
  int warp_tot[4];
};

// items of a tile: one uint16 per child, (record << 5) | slot, in child order, at items[lin * NQ_TILE * N ...]
// (one body over the record width R, one __global__ wrapper per width, as in nq_kernel.cuh; NqKernels below)
template <int N, int R>
__device__ __forceinline__ void nq_expand_count_body(const uint8_t* __restrict__ arena, const ExpandParams& prm,
                                                     uint16_t* __restrict__ items, int* __restrict__ tile_sums,
                                                     ExpandState* __restrict__ st) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  NqCountSmem<R>& sm = *reinterpret_cast<NqCountSmem<R>*>(smem_raw);
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  constexpr uint32_t IN_BYTES = NQ_TILE * R;
  const int first = blockIdx.x, stride = gridDim.x;
  if (t == 0) {
    mbar_init(&sm.full[0], 1);
    mbar_init(&sm.full[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  auto issue = [&](int lin, int s) {  // thread 0
    long long at, lo, hi;
    piece_of(prm, lin, NQ_TILE, at, lo, hi);
    const uint32_t nb = tile_load_bytes(at, hi, NQ_TILE, R);
    mbar_arrive_expect_tx(&sm.full[s], nb);
    if (nb) bulk_g2s(sm.in[s], arena + at * IN_BYTES, nb, &sm.full[s]);  // default L2 policy: the build kernel re-reads it
  };
  if (t == 0) {
    if (first < prm.n_tiles) issue(first, 0);
    if (first + stride < prm.n_tiles) issue(first + stride, 1);
  }
  unsigned my_solutions = 0;
  unsigned it = 0;
  for (int lin = first; lin < prm.n_tiles; lin += stride, it++) {
    const int s = it & 1;
    long long at, lo, hi;
    piece_of(prm, lin, NQ_TILE, at, lo, hi);
    mbar_wait(&sm.full[s], (it >> 1) & 1u);
    uint32_t cm[4];
    int leaves;
    nq_eval_quad<N, R>(sm.in[s], at * NQ_TILE, lo, hi, cm, leaves);
    // block scan of the child counts (leaves ride in the upper bits)
    const int mine = __popc(cm[0]) + __popc(cm[1]) + __popc(cm[2]) + __popc(cm[3]);
    int incl = mine | (leaves << 20);  // children of a tile <= 512*24 < 2^20
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) sm.warp_tot[wid] = incl;
    __syncthreads();  // everyone is done with in[s]; warp totals visible
    int woff = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      if (i < wid) woff += sm.warp_tot[i];
      tot += sm.warp_tot[i];
    }
    if (t == 0) {
      tile_sums[lin] = tot & 0xFFFFF;
      my_solutions += static_cast<unsigned>(tot >> 20);
      if (lin + 2 * stride < prm.n_tiles) issue(lin + 2 * stride, s);
    }
    uint16_t* gi = items + static_cast<long long>(lin) * (NQ_TILE * N) + (((woff + incl) & 0xFFFFF) - mine);
#pragma unroll
    for (int q = 0; q < 4; q++) {
      uint32_t m = cm[q];
      while (m) {
        const int k = __ffs(m) - 1;
        m &= m - 1;
        *gi++ = static_cast<uint16_t>(((4 * t + q) << 5) | k);
      }
    }
    __syncthreads();  // warp_tot free for the next tile
  }
  if (t == 0 && my_solutions) atomicAdd(&st->solutions, static_cast<unsigned long long>(my_solutions));
}
template <int N>
__global__ void __launch_bounds__(NQ_THREADS) nq_expand_count_kernel(const uint8_t* __restrict__ arena,
                                                                    const __grid_constant__ ExpandParams prm,
                                                                    uint16_t* __restrict__ items,
                                                                    int* __restrict__ tile_sums,
                                                                    ExpandState* __restrict__ st) {
  nq_expand_count_body<N, NQ_REC>(arena, prm, items, tile_sums, st);
}
template <int N>
__global__ void __launch_bounds__(NQ_THREADS) nq_expand_count_wide_kernel(const uint8_t* __restrict__ arena,
                                                                         const __grid_constant__ ExpandParams prm,
                                                                         uint16_t* __restrict__ items,
                                                                         int* __restrict__ tile_sums,
                                                                         ExpandState* __restrict__ st) {
  nq_expand_count_body<N, NQ_REC24>(arena, prm, items, tile_sums, st);
}

// ------------------------------------------------------------------------------------------- build
template <int R>
struct NqBuildSmem {
  alignas(128) uint8_t in[2][NQ_TILE * R];
  alignas(128) uint16_t item[2][EXP_CAP];  // first window of the tile's items
  alignas(128) uint8_t stage[EXP_CAP * R + 32];
  alignas(8) uint64_t full[2];             // one arrival per phase and load: parents, items
  alignas(8) uint64_t wbar;                // further item windows of dense tiles
  ScanSmem scan;
};

// child `c` of the tile -> bytes [B, B + R) of the staging image (B = image offset of the child).  The parent
// record sits at byte R*r of the tile (read at any alignment).
template <int R>
__device__ __forceinline__ void nq_build_child(const uint8_t* in_tile, int item, uint8_t* image, int B) {
  constexpr int W = nq_rec_words(R), L = W - 1;  // words of a record; the last one holds byte R - 1 only
  const int r = item >> 5, k = item & 31;
  const uint8_t* src = in_tile + r * R;
  // parent-aligned words: P[j] = parent bytes 4j .. 4j+3 (P[L]: byte R - 1 only)
  uint32_t P[W];
  nq_parent_words(src, P);
  P[L] &= 0xFFu;
  const uint32_t depth = P[0] & 0xFFu;
  // child = parent with depth+1 and board[depth] <=> board[k]: XOR both bytes with their difference
  const uint32_t p1 = 1u + depth, p2 = 1u + static_cast<uint32_t>(k);
  const uint32_t placed = src[p2];
  const uint32_t D = static_cast<uint32_t>(src[p1]) ^ placed;
  const uint32_t x1 = D << ((p1 & 3u) * 8u), x2 = D << ((p2 & 3u) * 8u);
  const uint32_t w1 = p1 >> 2, w2 = p2 >> 2;
#pragma unroll
  for (uint32_t j = 0; j < W; j++) P[j] ^= (j == w1 ? x1 : 0u) ^ (j == w2 ? x2 : 0u);
  P[0] += 1u;  // depth + 1 (depth < 255)
  // realign to the image: the child occupies bytes b .. b+R-1 of W aligned words
  const int b = B & 3;
  const uint32_t b8 = b * 8;
  uint32_t* dw = reinterpret_cast<uint32_t*>(image + (B - b));
  uint32_t Wd[W];
#pragma unroll
  for (int j = 0; j < W; j++) Wd[j] = shf_l_wrap(j ? P[j - 1] : 0u, P[j], b8);
#pragma unroll
  for (int j = 1; j < L; j++) dw[j] = Wd[j];
  // first and last word are shared with the neighbouring children: only this child's bytes
  uint8_t* d0 = reinterpret_cast<uint8_t*>(dw);
  if (b == 0) {
    dw[0] = Wd[0];
  } else {
    if (b <= 1) d0[1] = static_cast<uint8_t>(Wd[0] >> 8);
    if (b <= 2) d0[2] = static_cast<uint8_t>(Wd[0] >> 16);
    d0[3] = static_cast<uint8_t>(Wd[0] >> 24);
  }
  if (b == 3) {
    dw[L] = Wd[L];
  } else {
    d0[4 * L] = static_cast<uint8_t>(Wd[L]);
    if (b >= 1) d0[4 * L + 1] = static_cast<uint8_t>(Wd[L] >> 8);
    if (b >= 2) d0[4 * L + 2] = static_cast<uint8_t>(Wd[L] >> 16);
  }
}

// The same for a full warp of 32 consecutive children whose first one starts a word of the image (B = 4x for
// lane 0, hence B & 3 == lane & 3 as R = 1 mod 4): every word is stored whole — the word a child shares with its
// right-hand neighbour is completed with the neighbour's first bytes by a warp shuffle, lane 31 ends on a word
// boundary (32 * 21 bytes = 168 words, 32 * 25 = 200).  `active` = the child exists; all 32 lanes must call.
template <int R>
__device__ __forceinline__ void nq_build_child_warp(const uint8_t* in_tile, int item, uint8_t* image, int B,
                                                    bool active) {
  constexpr int W = nq_rec_words(R), L = W - 1;
  const int b = threadIdx.x & 3;
  const uint32_t b8 = b * 8;
  uint32_t W0 = 0, W1 = 0, W2 = 0, W3 = 0, W4 = 0, W5 = 0, W6 = 0;  // (W6: 25-byte records only)
  if (active) {
    const int r = item >> 5, k = item & 31;
    const uint8_t* src = in_tile + r * R;
    uint32_t P[W];
    nq_parent_words(src, P);
    P[L] &= 0xFFu;
    const uint32_t depth = P[0] & 0xFFu;
    const uint32_t p1 = 1u + depth, p2 = 1u + static_cast<uint32_t>(k);
    const uint32_t placed = src[p2];
    const uint32_t D = static_cast<uint32_t>(src[p1]) ^ placed;
    const uint32_t x1 = D << ((p1 & 3u) * 8u), x2 = D << ((p2 & 3u) * 8u);
    const uint32_t w1 = p1 >> 2, w2 = p2 >> 2;
#pragma unroll
    for (uint32_t j = 0; j < W; j++) P[j] ^= (j == w1 ? x1 : 0u) ^ (j == w2 ? x2 : 0u);
    P[0] += 1u;
    W0 = shf_l_wrap(0u, P[0], b8);
    W1 = shf_l_wrap(P[0], P[1], b8);
    W2 = shf_l_wrap(P[1], P[2], b8);
    W3 = shf_l_wrap(P[2], P[3], b8);
    W4 = shf_l_wrap(P[3], P[4], b8);
    W5 = shf_l_wrap(P[4], P[5], b8);
    if constexpr (L == 6) W6 = shf_l_wrap(P[5], P[L], b8);
  }
  const uint32_t nb = __shfl_down_sync(0xFFFFFFFFu, W0, 1);  // the right-hand neighbour's first word (0 if none)
  if (active) {
    uint32_t* dw = reinterpret_cast<uint32_t*>(image + (B - b));
    if (b == 0) dw[0] = W0;
    dw[1] = W1;
    dw[2] = W2;
    dw[3] = W3;
    dw[4] = W4;
    // (a last child writes up to 3 zero bytes past the image's end)
    if constexpr (L == 5) {
      dw[5] = b == 3 ? W5 : (W5 | nb);
    } else {
      dw[5] = W5;
      dw[6] = b == 3 ? W6 : (W6 | nb);
    }
  }
}

// (a kernel template over R itself: as a body behind per-width wrappers its 21-byte SASS would not stay the same)
template <int N, int R = NQ_REC>
__global__ void __launch_bounds__(NQ_THREADS) nq_expand_build_kernel(const uint8_t* __restrict__ arena,
                                                                    const __grid_constant__ ExpandParams prm,
                                                                    const uint16_t* __restrict__ items,
                                                                    const int* __restrict__ tile_sums,
                                                                    uint8_t* __restrict__ children,
                                                                    ExpandState* __restrict__ st,
                                                                    ExpandResult* __restrict__ res) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  NqBuildSmem<R>& sm = *reinterpret_cast<NqBuildSmem<R>*>(smem_raw);
  const int t = threadIdx.x;
  constexpr uint32_t IN_BYTES = NQ_TILE * R;
  constexpr long long IST = static_cast<long long>(NQ_TILE) * N;  // items per tile slot
  const int first = blockIdx.x, stride = gridDim.x;
  if (t == 0) {
    mbar_init(&sm.full[0], 2);
    mbar_init(&sm.full[1], 2);
    mbar_init(&sm.wbar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  uint64_t pol = 0;
  if (t == 0) pol = policy_evict_first();
  auto issue_parents = [&](int lin, int s) {  // thread 0
    long long at, lo, hi;
    piece_of(prm, lin, NQ_TILE, at, lo, hi);
    const uint32_t nb = tile_load_bytes(at, hi, NQ_TILE, R);
    mbar_arrive_expect_tx(&sm.full[s], nb);
    if (nb) bulk_g2s_stream(sm.in[s], arena + at * IN_BYTES, nb, &sm.full[s], pol);
  };
  auto issue_items = [&](int lin, int s, int cnt) {  // thread 0: the first window of the tile's items
    const uint32_t nb = (static_cast<uint32_t>(min(cnt, EXP_CAP)) * 2u + 15u) & ~15u;
    mbar_arrive_expect_tx(&sm.full[s], nb);
    if (nb) bulk_g2s_stream(sm.item[s], items + lin * IST, nb, &sm.full[s], pol);
  };
  if (t == 0) {  // the parents of the first two tiles are on their way while the offsets are computed
    if (first < prm.n_tiles) issue_parents(first, 0);
    if (first + stride < prm.n_tiles) issue_parents(first + stride, 1);
  }
  expand_own_offsets<NQ_THREADS>(sm.scan, tile_sums, prm.n_tiles, first, stride);
  expand_publish(sm.scan, st, res, prm.epoch, 0);
  if (t == 0) {
    if (first < prm.n_tiles) issue_items(first, 0, sm.scan.cnt[0]);
    if (first + stride < prm.n_tiles) issue_items(first + stride, 1, sm.scan.cnt[1]);
  }
  unsigned it = 0, wphase = 0;
  for (int lin = first; lin < prm.n_tiles; lin += stride, it++) {
    const int s = it & 1;
    const int total = sm.scan.cnt[it];
    uint8_t* const gtile = children + static_cast<long long>(sm.scan.own[it]) * R;
    mbar_wait(&sm.full[s], (it >> 1) & 1u);
    for (int c0 = 0; c0 < total; c0 += EXP_CAP) {  // windows of EXP_CAP children (one, except for dense tiles)
      const int cnt = min(EXP_CAP, total - c0);
      if (c0 > 0) {  // dense tile: fetch the next window of items (everyone passed (B) of the previous window)
        if (t == 0) {
          const uint32_t nb = (static_cast<uint32_t>(cnt) * 2u + 15u) & ~15u;
          mbar_arrive_expect_tx(&sm.wbar, nb);
          bulk_g2s_stream(sm.item[s], items + lin * IST + c0, nb, &sm.wbar, pol);
        }
        mbar_wait(&sm.wbar, wphase);
        wphase ^= 1u;
      }
      if (t == 0) bulk_wait_read<0>();  // the previous bulk store has drained the staging image
      __syncthreads();  // (A)
      uint8_t* gdst = gtile + static_cast<long long>(c0) * R;
      const int phase = static_cast<int>(reinterpret_cast<uintptr_t>(gdst) & 15);  // image and destination share it
      uint8_t* sdst = sm.stage + phase;
      // the first (-phase) & 3 children byte-wise, so that the warps' runs of 32 children start on a word
      const int c_head = min(cnt, (4 - (phase & 3)) & 3);
      if (t < c_head) nq_build_child<R>(sm.in[s], sm.item[s][t], sm.stage, phase + t * R);
      for (int cb = c_head; cb < cnt; cb += NQ_THREADS) {
        const int c = cb + t;
        const bool active = c < cnt;
        nq_build_child_warp<R>(sm.in[s], active ? sm.item[s][c] : 0, sm.stage, phase + c * R, active);
      }
      fence_async_smem();
      __syncthreads();  // (B) image complete; in[s] / item[s] free after the last window
      const int bytes = cnt * R;
      const int head = min(bytes, static_cast<int>((16 - (reinterpret_cast<uintptr_t>(gdst) & 15)) & 15));
      const int mid = (bytes - head) & ~15;
      const int tail = bytes - head - mid;
      if (t < head) gdst[t] = sdst[t];
      if (t >= 32 && t - 32 < tail) gdst[head + mid + (t - 32)] = sdst[head + mid + (t - 32)];
      if (t == 0 && mid > 0) {
        bulk_s2g(gdst + head, sdst + head, static_cast<uint32_t>(mid));
        bulk_commit();
      }
      // the head / tail bytes are read from the image after (B) by threads 1..47, which reach the next (A)
      // — after which the image is rewritten — only when they are done
    }
    // a tile without children has no barrier of its own: without this one thread 0 could re-arm full[s] twice
    // (tiles it+2, it+4) before a slow warp has tested the phase of tile it
    if (total == 0) __syncthreads();
    if (t == 0 && lin + 2 * stride < prm.n_tiles) {
      issue_parents(lin + 2 * stride, s);
      issue_items(lin + 2 * stride, s, sm.scan.cnt[it + 2]);
    }
  }
  if (t == 0) bulk_wait_all();
}

// the kernels of one record width: R = 21 (nq_*_kernel<N>) or 25 (nq_*_wide_kernel<N>; the build kernel: <N, R>)
template <int N, int R>
struct NqKernels;
template <int N>
struct NqKernels<N, NQ_REC> {
  static constexpr auto evaluate = nq_evaluate_kernel<N>;
  static constexpr auto evaluate_small = nq_evaluate_small_kernel<N>;
  static constexpr auto count = nq_expand_count_kernel<N>;
  static constexpr auto build = nq_expand_build_kernel<N, NQ_REC>;
};
template <int N>
struct NqKernels<N, NQ_REC24> {
  static constexpr auto evaluate = nq_evaluate_wide_kernel<N>;
  static constexpr auto evaluate_small = nq_evaluate_small_wide_kernel<N>;
  static constexpr auto count = nq_expand_count_wide_kernel<N>;
  static constexpr auto build = nq_expand_build_kernel<N, NQ_REC24>;
};

}  // namespace tsb

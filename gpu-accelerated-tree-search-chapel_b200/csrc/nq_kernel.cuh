// nq_kernel.cuh — N-Queens batch conflict check for sm_90a (H100).
//
// Replaces the reference's one-thread-per-(parent,k) foreach (nqueens_gpu_chpl.chpl:97-123;
// CUDA twin baselines/nqueens/nqueens_gpu_cuda.cu:137-164), which re-reads the 21-byte parent
// N times and runs an O(depth) loop per slot.  Here:
//   * the chunk is streamed through shared memory by the TMA engine (cp.async.bulk) in tiles of
//     512 parents (10 752 B in, 512*N B out), mbarrier pipeline, persistent CTAs;
//   * one thread owns FOUR consecutive parents = 84 B = 21 aligned words in, N aligned words out,
//     so the 21-byte / N-byte records never need unaligned or byte-wide memory instructions and
//     the word strides (21, N odd for N = 17, 19) are bank-conflict free;
//   * every kernel is a template over the record width R: 21 bytes (tsb_nq_node, MAX_QUEENS = 20) or 25 bytes
//     (tsb_nq_node24, a MAX_QUEENS = 24 build): four 25-byte parents are 25 aligned words, a tile 12 800 B.  Both
//     widths are 1 mod 4, which the byte-lane arithmetic of the child build (nq_expand.cuh) relies on;
//   * per parent the placed queens are folded once into a 32-bit "attacked values" mask U
//     (bit v set <=> value v is attacked on row `depth` by some placed queen), so
//     label[k] = !bit(U, board[k]): O(depth + N) per parent instead of O(depth * N).
//     Equivalent to the reference predicate (nqueens_gpu_chpl.chpl:112-118)
//         board[i] != board[k] - (depth-i)  &&  board[i] != board[k] + (depth-i)   for all i < depth
//     evaluated in int arithmetic (no uint8 wrap).
//
// The mask is built with ONE funnel shift per placed row.  For row i at distance s = depth - i
// let V_i be the 64-bit value with bits 32+s and 32-s set.  Then
//         high32( V_i << board[i] )  =  1 << (board[i] + s)  |  1 << (board[i] - s)
// with the out-of-range bits (>= 32 resp. < 0) falling off both ends by themselves — both
// diagonals, and the clamping, in one SHF.  The shift amount is taken in WRAP mode (low 5 bits
// of the register), so the raw packed word that holds board[i] in its low byte is used as the
// amount without extracting the byte (board values are < 32: a permutation of 0..N-1).
// V_i = (hi, lo) = (1 << s, 1 << (32-s)) is produced from two per-parent constants by constant
// shifts that make hi = lo = 0 for the rows i >= depth, so there are no per-row predicates.
// Labels are read back the same way: low32( (S << 8m) >> board[k] ) puts bit board[k] of the
// safe mask S = ~U at bit 8m, i.e. straight into byte m of the output word.
//
// Output contract: slots k >= depth are exact; slots k < depth are UNSPECIFIED, exactly as in the
// reference, whose kernel does not write them (nqueens_gpu_chpl.chpl:109,119) and whose consumer
// never reads them (:137-138).  `g` repeats an idempotent AND in the reference (:115-118); the
// result does not depend on it and the work is done once.
#pragma once
#include "xfer_route.h"
#include "tsb_ptx.cuh"

namespace tsb {

constexpr int NQ_THREADS = 128;
constexpr int NQ_QUAD = 4;                       // parents per thread
constexpr int NQ_TILE = NQ_THREADS * NQ_QUAD;    // 512 parents per tile
constexpr int NQ_REC = 21;                       // sizeof(tsb_nq_node)
constexpr int NQ_REC24 = 25;                     // sizeof(tsb_nq_node24)
constexpr int NQ_STAGES = 2;
// 32-bit words that hold an R-byte record starting at any byte of its first word (the last one holds one byte)
__host__ __device__ constexpr int nq_rec_words(int R) { return (R + 3) / 4; }

template <int N, int R = NQ_REC>
using NqSmem = TileSmem<NQ_STAGES, NQ_TILE * R, NQ_TILE * N>;

// Integer multiplies that must stay multiplies: they run on the FMA pipe (IMAD), which this
// kernel leaves idle, instead of the ALU pipe (SHF/LOP3), which is its bottleneck.
__device__ __forceinline__ uint32_t mul_lo_fma(uint32_t x, uint32_t c) {
  uint32_t r;
  asm("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(x), "r"(c));
  return r;
}

// a register whose LOW BYTE is byte B (compile-time) of the little-endian word array w
template <int B>
__device__ __forceinline__ uint32_t low_byte_reg(const uint32_t* w) {
  if constexpr ((B & 3) == 0)
    return w[B >> 2];
  else
    return w[B >> 2] >> (8 * (B & 3));
}

// rows [I0, I1) of parent Q: U |= OR_i high32(V_i << board[i])
template <int N, int I>
__device__ __forceinline__ uint32_t nq_row_term(uint32_t ph, uint32_t rb, const uint32_t (&amt)[N]) {
  if constexpr (I < N) {
    const uint32_t hi = mul_lo_fma(ph >> I, 2u);    // 1 << (depth - I) for I < depth, else 0
    const uint32_t lo = mul_lo_fma(rb, 1u << I);    // 1 << (32 - depth + I) for I < depth, else 0 (falls off)
    return shf_l_wrap(lo, hi, amt[I]);
  } else {
    return 0u;
  }
}
template <int N, int Q, int I0, int I1>
__device__ __forceinline__ void nq_rows(uint32_t ph, uint32_t rb, const uint32_t (&amt)[N], uint32_t& U) {
  static_assert(I1 - I0 == 4, "rows come in groups of four");
  U |= nq_row_term<N, I0>(ph, rb, amt) | nq_row_term<N, I0 + 1>(ph, rb, amt);
  U |= nq_row_term<N, I0 + 2>(ph, rb, amt) | nq_row_term<N, I0 + 3>(ph, rb, amt);
}

template <int N, int Q, int R = NQ_REC>
struct NqParent {
  static_assert(R % 4 == 1 && N < R, "records of 1 + 4k bytes, board values < 32");
  uint32_t depth, ph, rb, U;
  uint32_t amt[N];

  __device__ __forceinline__ void init(const uint32_t* w) {
    depth = low_byte_reg<R * Q>(w) & 0xFFu;
    ph = shl_clamp(1u, depth - 1u);   // 1 << (depth-1); 0 for depth == 0 (amount wraps to >= 32)
    rb = shl_clamp(1u, 32u - depth);  // 1 << (32-depth); 0 for depth == 0
    U = 0;
    fill_amt<0>(w);
  }
  template <int I>
  __device__ __forceinline__ void fill_amt(const uint32_t* w) {
    if constexpr (I < N) {
      amt[I] = low_byte_reg<R * Q + 1 + I>(w);
      fill_amt<I + 1>(w);
    }
  }
  template <int I0, int I1>
  __device__ __forceinline__ void rows() {
    nq_rows<N, Q, I0, I1>(ph, rb, amt, U);
  }
  // the safe-value mask S = ~U (N bits) pre-shifted to the four output byte lanes:
  // (S << 8m) as 64-bit (lo_m, hi_m) pairs; S < 2^24, so hi_0 = hi_1 = 0
  uint32_t lo_m[4], hi_m[4];
  __device__ __forceinline__ void finish_mask() {
    const uint32_t S = ~U & ((1u << N) - 1u);
    lo_m[0] = S;
    lo_m[1] = S << 8;
    lo_m[2] = S << 16;
    lo_m[3] = S << 24;
    hi_m[0] = 0u;
    hi_m[1] = 0u;
    hi_m[2] = S >> 16;
    hi_m[3] = S >> 8;
  }
  // slots [K0, K1): OR the label bits into the thread's output words
  template <int K0, int K1>
  __device__ __forceinline__ void slots(uint32_t (&o)[N]) {
#pragma unroll
    for (int k = K0; k < K1; k++) {
      if (k < N) {
        const int ob = Q * N + k;  // output byte index inside this thread's 4N bytes
        const int m = ob & 3;
        const uint32_t x = shf_r_wrap(lo_m[m], hi_m[m], amt[k]);
        o[ob >> 2] |= x & (1u << (8 * m));
      }
    }
  }
};

template <int N, int R>
__device__ __forceinline__ void nq_compute_tile(const uint8_t* in_tile, uint8_t* out_tile, int /*records*/) {
  const uint32_t* in_w = reinterpret_cast<const uint32_t*>(in_tile) + R * threadIdx.x;
  uint32_t* out_w = reinterpret_cast<uint32_t*>(out_tile) + N * threadIdx.x;
  uint32_t o[N];
#pragma unroll
  for (int i = 0; i < N; i++) o[i] = 0;

  NqParent<N, 0, R> p0;
  NqParent<N, 1, R> p1;
  NqParent<N, 2, R> p2;
  NqParent<N, 3, R> p3;
  uint32_t w[R];
#pragma unroll
  for (int i = 0; i < R; i++) w[i] = in_w[i];
  p0.init(w);
  p1.init(w);
  p2.init(w);
  p3.init(w);
  const uint32_t dmax = max(max(p0.depth, p1.depth), max(p2.depth, p3.depth));
  const uint32_t dmin = min(min(p0.depth, p1.depth), min(p2.depth, p3.depth));

  // rows in groups of 4, the four parents interleaved for ILP; a group is skipped when no parent
  // of this thread has placed queens in it (rows >= depth contribute nothing anyway)
#pragma unroll
  for (int j = 0; j < (N + 3) / 4; j++) {
    if (dmax > 4u * j) {
      switch (j) {  // compile-time row ranges
#define TSB_ROWS(J)                 \
  case J:                           \
    p0.template rows<4 * J, 4 * J + 4>(); \
    p1.template rows<4 * J, 4 * J + 4>(); \
    p2.template rows<4 * J, 4 * J + 4>(); \
    p3.template rows<4 * J, 4 * J + 4>(); \
    break;
        TSB_ROWS(0) TSB_ROWS(1) TSB_ROWS(2) TSB_ROWS(3) TSB_ROWS(4) TSB_ROWS(5)
#undef TSB_ROWS
      }
    }
  }
  p0.finish_mask();
  p1.finish_mask();
  p2.finish_mask();
  p3.finish_mask();
  // labels, again in groups of 4 slots; groups entirely below every parent's depth are skipped
  // (their slots are unspecified by contract)
#pragma unroll
  for (int j = 0; j < (N + 3) / 4; j++) {
    if (dmin < 4u * j + 4u) {
      switch (j) {
#define TSB_SLOTS(J)                 \
  case J:                            \
    p0.template slots<4 * J, 4 * J + 4>(o); \
    p1.template slots<4 * J, 4 * J + 4>(o); \
    p2.template slots<4 * J, 4 * J + 4>(o); \
    p3.template slots<4 * J, 4 * J + 4>(o); \
    break;
        TSB_SLOTS(0) TSB_SLOTS(1) TSB_SLOTS(2) TSB_SLOTS(3) TSB_SLOTS(4) TSB_SLOTS(5)
#undef TSB_SLOTS
      }
    }
  }
#pragma unroll
  for (int i = 0; i < N; i++) out_w[i] = o[i];
}

// Every kernel is a body over the record width R plus one __global__ wrapper per width: nq_*_kernel<N> (21 bytes)
// and nq_*_wide_kernel<N> (25 bytes, a MAX_QUEENS = 24 build); NqKernels<N, R> (nq_expand.cuh) names those of one
// width.
template <int N, int R>
__device__ __forceinline__ void nq_evaluate_body(const uint8_t* __restrict__ parents, uint8_t* __restrict__ labels,
                                                 long long count) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  NqSmem<N, R>& sm = *reinterpret_cast<NqSmem<N, R>*>(smem_raw);
  run_tile_pipeline<NQ_STAGES, NQ_TILE, R, N>(
      sm, parents, labels, count,
      [](const uint8_t* in_tile, uint8_t* out_tile, int n, long long) { nq_compute_tile<N, R>(in_tile, out_tile, n); });
}
template <int N>
__global__ void __launch_bounds__(NQ_THREADS) nq_evaluate_kernel(const uint8_t* __restrict__ parents,
                                                                uint8_t* __restrict__ labels, long long count) {
  nq_evaluate_body<N, NQ_REC>(parents, labels, count);
}
template <int N>
__global__ void __launch_bounds__(NQ_THREADS) nq_evaluate_wide_kernel(const uint8_t* __restrict__ parents,
                                                                     uint8_t* __restrict__ labels, long long count) {
  nq_evaluate_body<N, NQ_REC24>(parents, labels, count);
}

// ---- small chunks (the reference's default --M 50000 is 97 tiles of 512 parents: two thirds of the SMs, each thread
// working through four parents, behind a TMA pipeline set up for one tile): one parent per thread, 128 parents per
// CTA, plain coalesced 16-byte loads and stores — the shortest path from launch to labels.  The last CTA's bytes past
// its last whole 16-byte word are loaded one by one (nq_small_words, as the TMA path's partial tile): in zero-copy
// mode `parents` is the caller's registered host array, and nothing past its last record may be read.
template <int W>
__device__ __forceinline__ void nq_parent_words(const uint8_t* src, uint32_t (&P)[W]) {  // any byte alignment
  static_assert(W == 6 || W == 7, "21- or 25-byte records");
  const uint32_t mis = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src)) & 3u, a8 = mis * 8u;
  const uint32_t* sw = reinterpret_cast<const uint32_t*>(src - mis);
  const uint32_t s0 = sw[0], s1 = sw[1], s2 = sw[2], s3 = sw[3], s4 = sw[4], s5 = sw[5];
  P[0] = shf_r_wrap(s0, s1, a8);
  P[1] = shf_r_wrap(s1, s2, a8);
  P[2] = shf_r_wrap(s2, s3, a8);
  P[3] = shf_r_wrap(s3, s4, a8);
  P[4] = shf_r_wrap(s4, s5, a8);
  if constexpr (W == 6) {
    P[5] = shf_r_wrap(s5, 0u, a8);
  } else {
    const uint32_t s6 = sw[6];
    P[5] = shf_r_wrap(s5, s6, a8);
    P[6] = shf_r_wrap(s6, 0u, a8);
  }
}
constexpr int NQ_SMALL = 128;  // parents per CTA
template <int N, int R>
__device__ __forceinline__ void nq_evaluate_small_body(const uint8_t* __restrict__ parents, uint8_t* __restrict__ labels,
                                                       int count) {
  __shared__ __align__(16) uint8_t in[NQ_SMALL * R + 32];
  __shared__ __align__(16) uint8_t out[NQ_SMALL * N + 16];
  const int t = threadIdx.x;
  const int p0 = blockIdx.x * NQ_SMALL;
  const int np = min(NQ_SMALL, count - p0);
  {
    const uint8_t* src = parents + static_cast<size_t>(p0) * R;  // 128 * 21 = 168 * 16, 128 * 25 = 200 * 16: 16-byte aligned
    const int n16 = nq_small_words(np, R);
    for (int i = t; i < n16; i += NQ_SMALL) reinterpret_cast<uint4*>(in)[i] = reinterpret_cast<const uint4*>(src)[i];
    for (int i = 16 * n16 + t; i < np * R; i += NQ_SMALL) in[i] = src[i];
  }
  __syncthreads();
  if (t < np) {
    uint32_t P[nq_rec_words(R)];
    nq_parent_words(in + t * R, P);
    NqParent<N, 0, R> p;
    p.init(P);
    if (p.depth > 0u) p.template rows<0, 4>();
    if (p.depth > 4u) p.template rows<4, 8>();
    if (p.depth > 8u) p.template rows<8, 12>();
    if (p.depth > 12u) p.template rows<12, 16>();
    if (p.depth > 16u) p.template rows<16, 20>();
    if constexpr (N > 20) {
      if (p.depth > 20u) p.template rows<20, 24>();
    }
    const uint32_t S = ~p.U;
#pragma unroll
    for (int k = 0; k < N; k++) out[t * N + k] = static_cast<uint8_t>(shf_r_wrap(S, 0u, p.amt[k]) & 1u);
  }
  __syncthreads();
  uint8_t* dst = labels + static_cast<size_t>(p0) * N;  // 128 * N: a multiple of 16
  const int bytes = np * N, n16 = bytes >> 4;
  for (int i = t; i < n16; i += NQ_SMALL) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(out)[i];
  for (int i = 16 * n16 + t; i < bytes; i += NQ_SMALL) dst[i] = out[i];
}
template <int N>
__global__ void __launch_bounds__(NQ_SMALL) nq_evaluate_small_kernel(const uint8_t* __restrict__ parents,
                                                                    uint8_t* __restrict__ labels, int count) {
  nq_evaluate_small_body<N, NQ_REC>(parents, labels, count);
}
template <int N>
__global__ void __launch_bounds__(NQ_SMALL) nq_evaluate_small_wide_kernel(const uint8_t* __restrict__ parents,
                                                                         uint8_t* __restrict__ labels, int count) {
  nq_evaluate_small_body<N, NQ_REC24>(parents, labels, count);
}

}  // namespace tsb

// pfsp_kernels.cuh — PFSP lower bounds lb1 / lb1_d / lb2 over a chunk of parent nodes, sm_90a (H100).
//
// Reference kernels replaced: evaluate_gpu_lb1 (pfsp_gpu_chpl.chpl:192-208), evaluate_gpu_lb1_d
// (:216-235), evaluate_gpu_lb2 (:238-254) and the device math they call in
// lib/pfsp/Bound_simple.chpl / Bound_johnson.chpl.  The reference runs one thread per child
// slot (lb1, lb2), each of which re-copies the 88-byte parent and recomputes the parent's
// front/remain from scratch.  Here the chunk streams through shared memory by TMA bulk copies
// (tiles of 128 parents: 11 264 B in, 128*jobs*4 B out), the instance tables are staged into
// shared memory once per CTA by one bulk copy, and the prefix work shared by all children of a
// parent (front = completion times of the scheduled prefix, remain = unscheduled work per
// machine) is computed ONCE per parent:
//     child front   fc = add_forward(front, job)                (Bound_simple.chpl:29-35)
//     child remain  rc[j] = remain[j] - p[j][job]               (sum_unscheduled :94-106 on the child)
// which is exact integer arithmetic, so every bound is bit-identical to the reference.
#pragma once
#include <type_traits>

#include "tsb_ptx.cuh"

namespace tsb {

constexpr int PF_THREADS = 128;
constexpr int PF_TILE = 128;  // parents per tile (one per thread in the lb1 kernels)
constexpr int PF_REC = 88;    // sizeof(tsb_pfsp_node)
constexpr int PF_MAXJ = 20;
constexpr int PF_MAXM = 20;
constexpr int PF_MAXP = 190;

// Instance tables as staged into shared memory (one 16-B-multiple blob per handle).
struct PfspLb1Tables {
  int32_t jobs, machines, pairs, mp;   // mp = row stride of pj in ints (row_stride())
  int32_t total[PF_MAXM];              // sum_j p[k][j]
  int32_t min_heads[PF_MAXM];
  int32_t min_tails[PF_MAXM];
  int32_t pj[PF_MAXJ * 22];            // job-major: pj[job*mp + k], mp = row_stride(template M)
  uint32_t ph[PF_MAXJ * 12];           // the same rows with two machines per word (16 bits each):
                                       // ph[job*half_stride(M) + q] = p[2q][job] | p[2q+1][job] << 16
};
static_assert(sizeof(PfspLb1Tables) % 16 == 0, "blob must be a multiple of 16 B");
// the 16-bit lanes of ph and of the simd16 kernels: every intermediate of their bounds must stay below this
constexpr long long PF_LANE_LIMIT = 1 << 16;

__device__ __forceinline__ void stage_blob(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
    mbar_arrive_expect_tx(bar, bytes);
    bulk_g2s(dst_smem, src_gmem, bytes, bar);
  }
  __syncthreads();
  mbar_wait(bar, 0);
}

// ------------------------------------------------------------------------------------------- lb1 / lb1_d
// One thread per parent, 128 parents per tile.  Shared-memory traffic is the first bound of this
// kernel (every parent touches all 20 job rows of the processing-time table exactly once: the
// scheduled jobs in the front recurrence, the others as children), so every access is shaped to be
// bank-conflict free: node words are read as 11 x LDS.64 (stride 88 B = odd multiple of 8 B), job
// rows are `mp` ints at a stride of `mp` words read as LDS.64 (mp/2 odd for 10 machines), bounds
// are written as 5 x STS.128 (stride 80 B = odd multiple of 16 B).
// tiles: a ring of three 11 KB buffers used in place (run_tile_ring_inplace): the 80 B of bounds of a parent
// overwrite the tile once every thread holds its 88-byte node in registers -> 6 CTAs (24 warps) per SM with
// loads two tiles ahead (v4 had one input + one output buffer, 7 CTAs, and exposed the TMA wait).
struct Lb1Smem {
  RingSmem<PF_TILE * PF_REC> tiles;
  alignas(16) PfspLb1Tables tab;
  alignas(8) uint64_t tab_bar;
  int32_t bin[32];            // per-tile histogram of parent depths, then exclusive prefix
  uint8_t order[PF_TILE];     // parents of the tile sorted by depth
};

// Sort the parents of a tile by depth (counting sort in shared memory) and return the parent this
// thread should process.  The per-parent work grows with depth in the front recurrence and shrinks
// with it in the children loop, so a warp whose 32 parents have (nearly) the same depth executes
// close to the average number of steps instead of max-prefix + max-children of a mixed warp.
__device__ __forceinline__ int depth_sorted_parent(int32_t* bin, uint8_t* order, const uint8_t* in_tile,
                                                   int rec_lo, int rec_hi) {
  const int t = threadIdx.x;
  if (t < 32) bin[t] = 0;
  __syncthreads();
  int d = 31;  // records outside [rec_lo, rec_hi) sort last and stay idle
  if (t >= rec_lo && t < rec_hi) {
    d = reinterpret_cast<const int32_t*>(in_tile)[22 * t + 1] + 1;  // limit1 + 1 in 0..20
    d = min(max(d, 0), 30);
  }
  const int rank = atomicAdd(&bin[d], 1);
  __syncthreads();
  int base = 0;
  for (int b = 0; b < d; b++) base += bin[b];  // broadcast reads
  order[base + rank] = static_cast<uint8_t>(t);
  __syncthreads();
  return order[t];
}

// row stride (in ints) of the job-major table for a template machine count: ODD, so that the 20 job
// rows start in 20 different banks and a warp-wide 4-byte load of "machine k of each lane's job" is
// always one conflict-free wavefront (lanes with the same job broadcast).  8-byte row loads were
// measured at 1.6x the ideal wavefront count (16 bank pairs cannot hold 20 rows).
__host__ __device__ constexpr int row_stride(int M) { return M | 1; }

// row stride (in words) of the half-word packed table: odd as well
__host__ __device__ constexpr int half_words(int M) { return (M + 1) / 2; }
__host__ __device__ constexpr int half_stride(int M) { return half_words(M) | 1; }

// load row `job` of the job-major table: M machine times
template <int M>
__device__ __forceinline__ void load_row(const PfspLb1Tables& tab, int job, int (&row)[M]) {
  const int32_t* src = &tab.pj[job * row_stride(M)];
#pragma unroll
  for (int q = 0; q < M; q++) row[q] = src[q];
}

// integer add on the FMA pipe (IMAD): the max operations of the recurrences need the ALU pipe
__device__ __forceinline__ int add_fma(int a, int b) {
  int r;
  asm("mad.lo.s32 %0, %1, 1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}

// one scheduled job: front <- add_forward(front, job) (Bound_simple.chpl:29-35); remain -= p[.][job]
template <int M>
__device__ __forceinline__ void schedule_job(const PfspLb1Tables& tab, int job, int (&F)[M], int (&R)[M]) {
  int row[M];
  load_row<M>(tab, job, row);
  F[0] = add_fma(F[0], row[0]);
  R[0] = add_fma(R[0], -row[0]);
#pragma unroll
  for (int j = 1; j < M; j++) {
    F[j] = add_fma(max(F[j - 1], F[j]), row[j]);
    R[j] = add_fma(R[j], -row[j]);
  }
}

// front/remain of the parent's scheduled prefix prmu[0..limit1]  (schedule_front :47-62 +
// sum_unscheduled :94-106 rewritten as total - scheduled).  Generic form reading prmu from memory.
template <int M>
__device__ __forceinline__ void parent_front_remain(const PfspLb1Tables& tab, const int32_t* node, int limit1,
                                                    bool heads_if_root, int (&F)[M], int (&R)[M]) {
#pragma unroll
  for (int j = 0; j < M; j++) {
    F[j] = 0;
    R[j] = tab.total[j];
  }
  if (limit1 < 0) {
    if (heads_if_root) {
#pragma unroll
      for (int j = 0; j < M; j++) F[j] = tab.min_heads[j];
    }
    return;
  }
  for (int i = 0; i <= limit1; i++) schedule_job<M>(tab, node[2 + i], F, R);
}

// KIND 1: lb1_bound on the child (Bound_simple.chpl:123-136, machine_bound_from_parts :108-121)
// KIND 0: add_front_and_bound (Bound_simple.chpl:197-222)
template <int KIND, int M>
__device__ __forceinline__ int child_bound(const int (&F)[M], const int (&R)[M], const int (&B)[M],
                                           const int (&row)[M]) {
  if constexpr (KIND == 1) {
    // front_c[i] + remain_c[i] = (max(fc[i-1], F[i]) + p) + (R[i] - p) = max(fc[i-1], F[i]) + R[i]:
    // the child's own processing time cancels exactly (integers)
    int fc = add_fma(F[0], row[0]);  // child front, machine 0
    int tmp0 = F[0] + R[0];          // front_c[0] + remain_c[0]
    int lb = tmp0 + B[0];
#pragma unroll
    for (int i = 1; i < M; i++) {
      const int m = max(fc, F[i]);
      fc = add_fma(m, row[i]);
      const int tmp1 = max(tmp0, add_fma(m, R[i]));
      lb = __viaddmax_s32(tmp1, B[i], lb);  // max(lb, tmp1 + back[i])
      tmp0 = tmp1;
    }
    return lb;
  } else {
    // here R already holds remain[i] + back[i] (folded once per parent by the caller)
    int lb = F[0] + R[0];
    int tmp0 = add_fma(F[0], row[0]);
#pragma unroll
    for (int i = 1; i < M; i++) {
      const int tmp1 = max(tmp0, F[i]);
      lb = __viaddmax_s32(tmp1, R[i], lb);  // max(lb, tmp1 + remain[i] + back[i])
      tmp0 = add_fma(tmp1, row[i]);
    }
    return lb;
  }
}

// Two children at once in the two 16-bit halves of every register (DPX VIADDMNMX.U16x2 / VIMNMX.U16x2): the
// add_front_and_bound recurrence (Bound_simple.chpl:197-222)
//     lb = F[0] + RB[0];  t = F[0] + p[0];   for i >= 1:  s = max(t, F[i]);  lb = max(lb, s + RB[i]);  t = s + p[i]
// with RB = remain + back folded once per parent.  F2 / RB2 hold the parent's values in both halves; the
// children's processing times come from the half-word packed rows, one PRMT per machine interleaving the two
// jobs.  All values are < 2^16 (checked when the handle is created), so plain 32-bit adds never carry from
// the low half into the high one.  The lb1 entry point (lb1_bound on the child, Bound_simple.chpl:123-136)
// takes this route too when min_tails is non-increasing — then max_i(running max_j<=i a_j + back_i) =
// max_i(a_i + back_i), SURVEY.md Appendix A.4 — which fill_min_heads_tails guarantees; otherwise, and for values
// beyond 16 bits, the scalar formulation above is used.
template <int M>
__device__ __forceinline__ uint32_t child_pair_bound(const PfspLb1Tables& tab, const uint32_t (&F2)[M],
                                                     const uint32_t (&RB2)[M], int job_a, int job_b) {
  constexpr int HW = half_words(M);
  const uint32_t* ra = &tab.ph[job_a * half_stride(M)];
  const uint32_t* rb = &tab.ph[job_b * half_stride(M)];
  uint32_t wa[HW], wb[HW];
#pragma unroll
  for (int q = 0; q < HW; q++) {
    wa[q] = ra[q];
    wb[q] = rb[q];
  }
  uint32_t lb = F2[0] + RB2[0];
  uint32_t t = F2[0] + __byte_perm(wa[0], wb[0], 0x5410);  // + (p_a[0], p_b[0])
#pragma unroll
  for (int i = 1; i < M; i++) {
    const uint32_t s = __vmaxu2(t, F2[i]);
    lb = __viaddmax_u16x2(s, RB2[i], lb);
    const uint32_t p2 = __byte_perm(wa[i >> 1], wb[i >> 1], (i & 1) ? 0x7632 : 0x5410);
    t = s + p2;
  }
  return lb;
}

// Bounds of all children of the tile's parents [rec_lo, rec_hi).  `emit(t, limit1, g, v)` receives, for parent
// t and every group g of four slots with at least one live slot (k = 4g..4g+3 > limit1), the four bounds.
// Returns the record this thread was given by the depth sort (a permutation of the tile's 128 records).
template <int KIND, int M, bool SIMD, bool INPLACE, typename Emit>
__device__ __forceinline__ int lb1_compute_tile(Lb1Smem& sm, const uint8_t* in_tile, int rec_lo, int rec_hi,
                                                Emit&& emit) {
  const PfspLb1Tables& tab = sm.tab;
  const int t = depth_sorted_parent(sm.bin, sm.order, in_tile, rec_lo, rec_hi);
  const bool valid = t >= rec_lo && t < rec_hi;
  // the node: 22 ints as 11 8-byte loads
  const int2* node2 = reinterpret_cast<const int2*>(in_tile) + 11 * t;
  int prmu[PF_MAXJ];
  const int2 head = node2[0];
  const int limit1 = min(max(head.y, -1), PF_MAXJ - 1);
#pragma unroll
  for (int q = 0; q < 10; q++) {
    const int2 v = node2[1 + q];
    prmu[2 * q] = valid ? v.x : 0;
    prmu[2 * q + 1] = valid ? v.y : 0;
  }
  if constexpr (INPLACE) __syncthreads();  // every node is in registers: emit() may overwrite the tile
  if (!valid) return t;
  int F[M], R[M], B[M];
#pragma unroll
  for (int j = 0; j < M; j++) {
    F[j] = 0;
    R[j] = tab.total[j];
    B[j] = tab.min_tails[j];  // schedule_back with limit2 == jobs (:70-74)
  }
  if (KIND == 0 && limit1 < 0) {  // lb1_d on the root: front = min_heads (schedule_front :53-57)
#pragma unroll
    for (int j = 0; j < M; j++) F[j] = tab.min_heads[j];
  }
  // two scheduled jobs per step: the second job's chain can start one machine behind the first
  // one's (wavefront parallelism) when both sit in one branch-free block
#pragma unroll
  for (int i = 0; i < PF_MAXJ; i += 2) {
    if (i > limit1) break;
    if (i + 1 <= limit1) {
      int r0[M], r1[M];
      load_row<M>(tab, prmu[i], r0);
      load_row<M>(tab, prmu[i + 1], r1);
      int f0 = add_fma(F[0], r0[0]);
      int f1 = add_fma(f0, r1[0]);
      R[0] = R[0] - r0[0] - r1[0];  // one three-input add (the kernel is issue-bound, not ALU-pipe-bound)
      F[0] = f1;
#pragma unroll
      for (int j = 1; j < M; j++) {
        f0 = add_fma(max(f0, F[j]), r0[j]);  // job i on machine j
        f1 = add_fma(max(f1, f0), r1[j]);    // job i+1 on machine j
        R[j] = R[j] - r0[j] - r1[j];
        F[j] = f1;
      }
    } else {
      schedule_job<M>(tab, prmu[i], F, R);
    }
  }
  if constexpr (SIMD) {
    uint32_t F2[M], RB2[M];
#pragma unroll
    for (int j = 0; j < M; j++) {
      F2[j] = static_cast<uint32_t>(F[j]) * 0x10001u;
      RB2[j] = static_cast<uint32_t>(R[j] + B[j]) * 0x10001u;
    }
    // children in groups of four slots = two pairs; a pair with no live slot is skipped
#pragma unroll
    for (int g = 0; g < 5; g++) {
      if (4 * g + 3 > limit1) {
        int v[4] = {0, 0, 0, 0};
        if (4 * g + 1 > limit1) {
          const uint32_t x = child_pair_bound<M>(tab, F2, RB2, prmu[4 * g], prmu[4 * g + 1]);
          v[0] = static_cast<int>(x & 0xFFFFu);
          v[1] = static_cast<int>(x >> 16);
        }
        const uint32_t y = child_pair_bound<M>(tab, F2, RB2, prmu[4 * g + 2], prmu[4 * g + 3]);
        v[2] = static_cast<int>(y & 0xFFFFu);
        v[3] = static_cast<int>(y >> 16);
        emit(t, limit1, g, v);
      }
    }
    return t;
  }
  if constexpr (KIND == 0) {  // fold remain + back once per parent
#pragma unroll
    for (int j = 0; j < M; j++) R[j] += B[j];
  }
  // children in groups of four slots.  A group with at least one live slot evaluates all four slots without
  // branches (four independent recurrences to interleave); the values of slots k <= limit1 are unspecified
  // by contract.
#pragma unroll
  for (int g = 0; g < 5; g++) {
    if (4 * g + 3 > limit1) {
      int v[4];
#pragma unroll
      for (int c = 0; c < 4; c++) {
        int row[M];
        load_row<M>(tab, prmu[4 * g + c], row);
        v[c] = child_bound<KIND, M>(F, R, B, row);
      }
      emit(t, limit1, g, v);
    }
  }
  return t;
}

template <int KIND, int M, bool SIMD>
__global__ void __launch_bounds__(PF_THREADS) pfsp_lb1_kernel(const uint8_t* __restrict__ parents,
                                                             uint8_t* __restrict__ bounds, long long count,
                                                             const PfspLb1Tables* __restrict__ tables) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  Lb1Smem& sm = *reinterpret_cast<Lb1Smem*>(smem_raw);
  stage_blob(&sm.tab, tables, sizeof(PfspLb1Tables), &sm.tab_bar);
  run_tile_ring_inplace<PF_TILE, PF_REC, PF_MAXJ * 4>(
      sm.tiles, parents, bounds, count, [&sm](uint8_t* tile, int n, long long) {
        // one 16-byte store per group of four slots (stride 80 B = odd multiple of 16 B: conflict free)
        lb1_compute_tile<KIND, M, SIMD, true>(sm, tile, 0, n, [tile](int t, int, int g, const int (&v)[4]) {
          reinterpret_cast<int4*>(tile)[5 * t + g] = make_int4(v[0], v[1], v[2], v[3]);
        });
      });
}

// ------------------------------------------------------------------------------------------- lb2
// lb2_bound (Bound_johnson.chpl:274-289): front/back as above, flags of scheduled jobs
// (set_flags :179-186, here a 20-bit register mask), then lb_makespan (:214-240) over the
// machine pairs in machine_pair_order with compute_cmax_johnson (:188-212) per pair and the
// early exit `lb > best` reproduced exactly (first pair, in order, where the running max
// exceeds best).
//
// v2.  The Johnson tables are PACKED and live in the constant bank (kernel parameter): one word per
// (pair, position) = job | p[ma0][job] << 5 | p[ma1][job] << 12 | lag << 19 and one word per pair
// = ma0 | ma1 << 5 | min_tails[ma0] << 10 | min_tails[ma1] << 21, both in machine_pair_order.  All lanes
// of a warp walk the same (pair, position), so the table word is a uniform constant load and its
// unpacking runs on the uniform datapath; per lane and position only the scheduled-bit test, two adds and
// one max remain (v1: four dependent shared-memory loads per position and 34 KB of tables per CTA).
// Per tile of 64 parents: (A) one thread per parent computes the parent front and appends its live
// (parent, slot) children to a shared list; (B) the pairs are processed in chunks of LB2_CHUNK: every
// thread takes children from the ACTIVE list, rebuilds the child front (10 adds), runs the chunk, and
// re-appends the child to the next list unless its bound already exceeds `best` — about 90 % of the
// children are pruned within the first pairs, and compacting the survivors keeps the warps full (v1 kept
// a whole warp busy for all pairs as soon as one of its 32 children survived).
#ifndef TSB_LB2_TILE
#define TSB_LB2_TILE 64
#endif
#ifndef TSB_LB2_CHUNK
#define TSB_LB2_CHUNK 9
#endif
constexpr int LB2_TILE = TSB_LB2_TILE;
constexpr int LB2_STAGES = 2;
constexpr int LB2_CHUNK = TSB_LB2_CHUNK;  // machine pairs between two compactions
struct Lb2Const {
  uint32_t pair[PF_MAXP + 2];
  uint32_t jp[PF_MAXP * PF_MAXJ];
};
static_assert(sizeof(Lb2Const) <= 16 * 1024, "must fit the kernel parameter space next to the other arguments");
// The words of Lb2Const, decoded in lb2_phase_b (Lb2Const) (the pair words of pfsp_wide.cuh too).  Instances whose values do
// not fit these fields get no lb2.
//   pair word: ma0 | ma1 << 5 | min_tails[ma0] << 10 | min_tails[ma1] << 21
//   job word:  job | p[ma0][job] << 5 | p[ma1][job] << 12 | lag << 19
constexpr uint32_t LB2_MACH_MASK = 31, LB2_TAIL_MAX = 2047;
constexpr int LB2_MB_SHIFT = 5, LB2_TA_SHIFT = 10, LB2_TB_SHIFT = 21;
constexpr uint32_t LB2_JOB_MASK = 31, LB2_P_MAX = 127, LB2_LAG_MAX = 8191;
constexpr int LB2_PA_SHIFT = 5, LB2_PB_SHIFT = 12, LB2_LAG_SHIFT = 19;
static_assert(LB2_TB_SHIFT + 11 == 32 && LB2_LAG_SHIFT + 13 == 32, "the top field of a word is read without a mask");
inline bool lb2_fits(int v, uint32_t max) { return v >= 0 && static_cast<uint32_t>(v) <= max; }
inline uint32_t lb2_pair_word(int a, int b, int tail_a, int tail_b) {
  return static_cast<uint32_t>(a) | static_cast<uint32_t>(b) << LB2_MB_SHIFT |
         (static_cast<uint32_t>(tail_a) & LB2_TAIL_MAX) << LB2_TA_SHIFT |
         (static_cast<uint32_t>(tail_b) & LB2_TAIL_MAX) << LB2_TB_SHIFT;
}
inline uint32_t lb2_job_word(int job, int pa, int pb, int lag) {
  return static_cast<uint32_t>(job) | (static_cast<uint32_t>(pa) & LB2_P_MAX) << LB2_PA_SHIFT |
         (static_cast<uint32_t>(pb) & LB2_P_MAX) << LB2_PB_SHIFT | (static_cast<uint32_t>(lag) & LB2_LAG_MAX) << LB2_LAG_SHIFT;
}
// v3, for instances with at most 10 machines (45 pairs) whose values fit 16 bits: one table word per USE (nothing
// is unpacked) and the Johnson recurrence of a pair (compute_cmax_johnson, Bound_johnson.chpl:188-212)
//     t0 += p0[j];   t1 = max(t1, t0 + lag[j]) + p1[j]        over the unscheduled jobs j in Johnson order
// rewritten in closed max-plus form.  With A_j = sum_{i<=j} p0[i], B_j = sum_{i<j} p1[i] over the unscheduled jobs,
//     t0_final = t0 + S0,      t1_final = S1 + max(t1, t0 + max_j (A_j - B_j + lag[j]))
// where S0, S1 = the child's remaining work on the two machines (known per child: remain - its own job).  Exact in
// integers, and the per-position work becomes two INDEPENDENT one-instruction chains
//     D = E + c1[j];  m = max(m, D);  E += c2[j]        c1 = p0 + lag,  c2 = p0 - p1
// instead of one three-instruction dependent chain — the kernel is latency-bound on that chain, not issue-bound
// (a fully unrolled pair loop with half the instructions ran no faster, and slower from 280 KB of code).
// The constant bank turned out to be the wrong home for one-word-per-use tables (three LDC per position cost more
// than the unpacking they save), so for <= 10 machines the table lives in SHARED memory as one uint4 per
// (pair, position) = {1 << job, c1, c2, 0}: a single broadcast LDS.128 per position, no unpacking, four ALU-pipe
// instructions (scheduled-bit test, add, max, add).
constexpr int LB2U_PAIRS = 45;
struct Lb2TabU {
  uint4 e[LB2U_PAIRS * PF_MAXJ];  // {bit, c1 = p[ma0] + lag, c2 = p[ma0] - p[ma1], 0} in machine_pair_order / Johnson order
  uint32_t mach[LB2U_PAIRS + 3];  // ma0 | ma1 << 8
  uint32_t tails[LB2U_PAIRS + 3]; // min_tails[ma0] | min_tails[ma1] << 16
};
static_assert(sizeof(Lb2TabU) % 16 == 0, "blob must be a multiple of 16 B");
// the entries of Lb2TabU, decoded in lb2_phase_b (Lb2ConstU); values fit 16 bits (the simd16 route's condition)
constexpr int LB2U_MB_SHIFT = 8, LB2U_TB_SHIFT = 16;
inline uint32_t lb2u_mach_word(int a, int b) { return static_cast<uint32_t>(a) | static_cast<uint32_t>(b) << LB2U_MB_SHIFT; }
inline uint32_t lb2u_tails_word(int tail_a, int tail_b) {
  return static_cast<uint32_t>(tail_a) | static_cast<uint32_t>(tail_b) << LB2U_TB_SHIFT;
}
inline uint4 lb2u_entry(int job, int pa, int pb, int lag) {
  return make_uint4(1u << job, static_cast<uint32_t>(pa + lag), static_cast<uint32_t>(pa - pb), 0u);
}
struct Lb2ConstU {  // kernel-parameter form of the route: just the device address of the table
  const Lb2TabU* tab;
};
using Lb2Tiles = TileSmem<LB2_STAGES, LB2_TILE * PF_REC, LB2_TILE * PF_MAXJ * 4>;

struct Lb2TabNone {
  uint4 e[1];
  uint32_t mach[4], tails[4];
};
template <int M>
struct Lb2TabSlot {
  using type = typename std::conditional<(M <= 10), Lb2TabU, Lb2TabNone>::type;
};
template <int M>
struct Lb2Smem {
  Lb2Tiles tiles;
  alignas(16) PfspLb1Tables tab1;
  alignas(8) uint64_t tab_bar[2];
  int32_t front[M][LB2_TILE];                   // parent fronts, [machine][parent]
  int32_t remain[M][LB2_TILE];                  // parent remaining work, [machine][parent]
  int32_t fc[M][PF_THREADS];                    // per-thread child front scratch, [machine][thread]
  int32_t rc[M][PF_THREADS];                    // per-thread child remaining work
  alignas(16) typename Lb2TabSlot<M>::type tabu;  // the Lb2ConstU route's table (M <= 10 only)
  uint32_t sched[LB2_TILE];                     // bit j set <=> job j scheduled in the parent
  uint32_t list[2][LB2_TILE * PF_MAXJ];         // active children: parent << 24 | slot << 16 | running lb
  int32_t n_list[2];
};

// child front = add_forward(parent front, job) into this thread's column of sm.fc; returns the scheduled mask
template <int M>
__device__ __forceinline__ uint32_t lb2_child_front(Lb2Smem<M>& sm, const int32_t* nodes, int p, int k) {
  const int t = threadIdx.x;
  const PfspLb1Tables& tab = sm.tab1;
  const int job = nodes[22 * p + 2 + k];
  int row[M];
  load_row<M>(tab, job, row);
  int f = sm.front[0][p] + row[0];
  sm.fc[0][t] = f;
  sm.rc[0][t] = sm.remain[0][p] - row[0];
#pragma unroll
  for (int j = 1; j < M; j++) {
    f = max(f, sm.front[j][p]) + row[j];
    sm.fc[j][t] = f;
    sm.rc[j][t] = sm.remain[j][p] - row[j];
  }
  return sm.sched[p] | (1u << job);
}

// instance tables -> shared memory (one or two bulk copies on one barrier)
template <int M>
__device__ __forceinline__ void lb2_stage_tables(Lb2Smem<M>& sm, const PfspLb1Tables* tables1, const Lb2Const&) {
  stage_blob(&sm.tab1, tables1, sizeof(PfspLb1Tables), &sm.tab_bar[0]);
}
template <int M>
__device__ __forceinline__ void lb2_stage_tables(Lb2Smem<M>& sm, const PfspLb1Tables* tables1, const Lb2ConstU& C) {
  if (threadIdx.x == 0) {
    mbar_init(&sm.tab_bar[0], 1);
    mbar_fence_init();
    mbar_arrive_expect_tx(&sm.tab_bar[0], sizeof(PfspLb1Tables) + (M <= 10 ? sizeof(Lb2TabU) : 0));
    bulk_g2s(&sm.tab1, tables1, sizeof(PfspLb1Tables), &sm.tab_bar[0]);
    if constexpr (M <= 10) bulk_g2s(&sm.tabu, C.tab, sizeof(Lb2TabU), &sm.tab_bar[0]);
  }
  __syncthreads();
  mbar_wait(&sm.tab_bar[0], 0);
}

// ---- phase B, packed tables, rolled pair loop (any machine count)
template <int M, typename Emit>
__device__ __forceinline__ void lb2_phase_b(Lb2Smem<M>& sm, const Lb2Const& C, const int32_t* nodes, int best,
                                            Emit&& emit) {
  const int t = threadIdx.x;
  const int pairs = sm.tab1.pairs;
  int cur = 0;
  for (int l0 = 0; l0 < pairs; l0 += LB2_CHUNK, cur ^= 1) {
    const int n_act = sm.n_list[cur];
    if (n_act == 0) break;  // (uniform)
    const int l1 = min(pairs, l0 + LB2_CHUNK);
    const bool last = l1 == pairs;
    for (int it = t; it < n_act; it += PF_THREADS) {
      const uint32_t e = sm.list[cur][it];
      const int p = e >> 24, k = (e >> 16) & 31;
      int lb = e & 0xFFFF;
      const uint32_t mask = lb2_child_front<M>(sm, nodes, p, k);
      bool over = false;
      for (int l = l0; l < l1; l++) {
        const uint32_t pi = C.pair[l];
        int tmp0 = sm.fc[pi & LB2_MACH_MASK][t], tmp1 = sm.fc[(pi >> LB2_MB_SHIFT) & LB2_MACH_MASK][t];
        const uint32_t* jp = &C.jp[l * PF_MAXJ];
#pragma unroll
        for (int j = 0; j < PF_MAXJ; j++) {
          const uint32_t w = jp[j];
          if (!(mask & (1u << (w & LB2_JOB_MASK)))) {
            tmp0 += static_cast<int>((w >> LB2_PA_SHIFT) & LB2_P_MAX);
            tmp1 = max(tmp1, tmp0 + static_cast<int>(w >> LB2_LAG_SHIFT)) + static_cast<int>((w >> LB2_PB_SHIFT) & LB2_P_MAX);
          }
        }
        const int c = max(tmp1 + static_cast<int>(pi >> LB2_TB_SHIFT), tmp0 + static_cast<int>((pi >> LB2_TA_SHIFT) & LB2_TAIL_MAX));
        lb = max(lb, c);
        if (lb > best) {
          over = true;
          break;
        }
      }
      if (over || last) {
        emit(p, k, lb);
      } else {
        const int at = atomicAdd(&sm.n_list[cur ^ 1], 1);
        sm.list[cur ^ 1][at] = (e & 0xFFFF0000u) | static_cast<uint32_t>(lb);
      }
    }
    __syncthreads();
    if (t == 0) sm.n_list[cur] = 0;  // becomes the "next" list of the following chunk
    __syncthreads();
  }
}

// ---- phase B, one-word-per-use tables (Lb2ConstU): pairs rolled, the 20 positions unrolled
// (a fully unrolled pair loop — 45 x 20 positions, every table word an immediate-address constant load — was
// measured SLOWER than this: 280 KB of code per kernel)
template <int M, typename Emit>
__device__ __forceinline__ void lb2_phase_b(Lb2Smem<M>& sm, const Lb2ConstU&, const int32_t* nodes, int best,
                                            Emit&& emit) {
  const int t = threadIdx.x;
  const int pairs = sm.tab1.pairs;
  int cur = 0;
  for (int l0 = 0; l0 < pairs; l0 += LB2_CHUNK, cur ^= 1) {
    const int n_act = sm.n_list[cur];
    if (n_act == 0) break;  // (uniform)
    const int l1 = min(pairs, l0 + LB2_CHUNK);
    const bool last = l1 == pairs;
    for (int it = t; it < n_act; it += PF_THREADS) {
      const uint32_t e = sm.list[cur][it];
      const int p = e >> 24, k = (e >> 16) & 31;
      int lb = e & 0xFFFF;
      const uint32_t mask = lb2_child_front<M>(sm, nodes, p, k);
      bool over = false;
      for (int l = l0; l < l1; l++) {
        const uint32_t mm = sm.tabu.mach[l];
        const int ma0 = mm & ((1u << LB2U_MB_SHIFT) - 1), ma1 = mm >> LB2U_MB_SHIFT;
        const uint4* te = &sm.tabu.e[l * PF_MAXJ];
        int E = 0, m = -(1 << 28);
#pragma unroll
        for (int j = 0; j < PF_MAXJ; j++) {
          const uint4 w = te[j];  // broadcast LDS.128
          if (!(mask & w.x)) {
            m = max(m, E + static_cast<int>(w.y));
            E += static_cast<int>(w.z);
          }
        }
        const uint32_t tl = sm.tabu.tails[l];
        const int t0 = sm.fc[ma0][t];
        const int t1f = sm.rc[ma1][t] + max(sm.fc[ma1][t], t0 + m);
        const int c = max(t1f + static_cast<int>(tl >> LB2U_TB_SHIFT),
                          t0 + sm.rc[ma0][t] + static_cast<int>(tl & ((1u << LB2U_TB_SHIFT) - 1)));
        lb = max(lb, c);
        if (lb > best) {
          over = true;
          break;
        }
      }
      if (over || last) {
        emit(p, k, lb);
      } else {
        const int at = atomicAdd(&sm.n_list[cur ^ 1], 1);
        sm.list[cur ^ 1][at] = (e & 0xFFFF0000u) | static_cast<uint32_t>(lb);
      }
    }
    __syncthreads();
    if (t == 0) sm.n_list[cur] = 0;
    __syncthreads();
  }
}

// `emit(p, k, lb)` receives the bound of every live (parent p, slot k) of the tile's parents [rec_lo, rec_hi);
// `dead(p, k)` is called for the slots below the live range (the evaluator zeroes them).
template <int M, typename CT, typename Emit, typename Dead>
__device__ __forceinline__ void lb2_compute_tile(Lb2Smem<M>& sm, const CT& C, const uint8_t* in_tile, int rec_lo,
                                                 int rec_hi, int best, Emit&& emit, Dead&& dead) {
  const int t = threadIdx.x;
  const PfspLb1Tables& tab = sm.tab1;
  const int jobs = tab.jobs;
  const int32_t* nodes = reinterpret_cast<const int32_t*>(in_tile);

  if (t < 2) sm.n_list[t] = 0;
  __syncthreads();
  // ---- phase A
  if (t < LB2_TILE && t >= rec_lo && t < rec_hi) {
    const int32_t* node = nodes + 22 * t;
    const int limit1 = min(max(node[1], -1), PF_MAXJ - 1);
    int F[M], R[M];
    parent_front_remain<M>(tab, node, limit1, false, F, R);  // lb2 children always have limit1 >= 0
#pragma unroll
    for (int j = 0; j < M; j++) {
      sm.front[j][t] = F[j];
      sm.remain[j][t] = R[j];
    }
    uint32_t mask = 0;
    for (int i = 0; i <= limit1; i++) mask |= 1u << node[2 + i];
    sm.sched[t] = mask;
    const int live = jobs - 1 - limit1;
    int base = live > 0 ? atomicAdd(&sm.n_list[0], live) : 0;
    for (int k = 0; k < jobs; k++) {
      if (k > limit1)
        sm.list[0][base++] = (static_cast<uint32_t>(t) << 24) | (static_cast<uint32_t>(k) << 16);
      else
        dead(t, k);
    }
  }
  __syncthreads();
  lb2_phase_b<M>(sm, C, nodes, best, emit);
}

template <int M, typename CT>
__global__ void __launch_bounds__(PF_THREADS) pfsp_lb2_kernel(const uint8_t* __restrict__ parents,
                                                             uint8_t* __restrict__ bounds, long long count,
                                                             const PfspLb1Tables* __restrict__ tables1,
                                                             const __grid_constant__ CT C, int best) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  Lb2Smem<M>& sm = *reinterpret_cast<Lb2Smem<M>*>(smem_raw);
  lb2_stage_tables(sm, tables1, C);
  run_tile_pipeline<LB2_STAGES, LB2_TILE, PF_REC, PF_MAXJ * 4>(
      sm.tiles, parents, bounds, count, [&sm, &C, best](const uint8_t* in_tile, uint8_t* out_tile, int n, long long) {
        int32_t* out = reinterpret_cast<int32_t*>(out_tile);
        const int jobs = sm.tab1.jobs;
        lb2_compute_tile<M>(
            sm, C, in_tile, 0, n, best, [out, jobs](int p, int k, int lb) { out[jobs * p + k] = lb; },
            [out, jobs](int p, int k) { out[jobs * p + k] = 0; });
      });
}

}  // namespace tsb

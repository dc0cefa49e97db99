// pfsp_rounds.cuh — the persistent multi-round PFSP kernel (lb1 / lb1_d), sm_90a (H100).
//
// The PFSP twin of nq_rounds_ll.cuh: the whole offload loop of pfsp_gpu_chpl.chpl:376-392 (popBackBulk(m, M),
// evaluate_gpu, generate_children, round after round) in ONE cooperative launch instead of two kernels and a host
// round trip per round (tsb_pfsp_pool_step).  While the kernel runs, the pool is one contiguous stack [0, size) of
// 88-byte records in the arena (the host compacts it before the launch).  Every CTA tracks the pool state (size,
// epoch, counters, exit decision) redundantly from the round totals, which every CTA gathers anyway, so nothing is
// broadcast.  A round:
//   (1) exit tests (uniform): DONE (size < m), PAUSE (max_rounds), SPACE (the worst case size - n + n * jobs does not
//       fit the arena); else the chunk is the top n = min(size, M) records, cut into 2G equal sub-slices: CTA k takes
//       number k from the bottom and number k from the top (the bottom of a chunk holds the shallow nodes, which have
//       the most children to evaluate and store; pairing evens the load, as in nq_rounds_ll.cuh)
//   (2) the slice -> shared memory (L2 loads: the records were stored by other CTAs in the previous round)
//   (3) child masks, leaf count and leaf minimum of the slice, 128 parents at a time, by the bound code of the count
//       kernel (lb1_compute_tile, pfsp_kernels.cuh; pfsp_expand_count_lb1_kernel's epilogue)
//   (4) COUNT EXCHANGE: the CTA publishes {children, leaves, leaf minimum} in its epoch-tagged slot, builds its child
//       list (record, slot) in shared memory, and gathers every slot.  A CTA publishes only after its whole slice
//       is in shared memory, so seeing every slot proves that every slice of the chunk has been read: the children
//       may overwrite the chunk in place (the argument of nq_rounds_ll.cuh's count exchange)
//   (5) IMPROVED (uniform, before any store): the chunk's leaf minimum is below `best`.  The reference's
//       generate_children lowers best while it walks the chunk, which changes what the rest of the chunk pushes; the
//       round is NOT committed (nothing stored, counts dropped) and the kernel leaves, so that the host runs that one
//       round through tsb_pfsp_pool_step (whose slow path applies the sequential rule) and relaunches with the new
//       best.  With --ub 1 (best = optimum) this never happens.
//   (6) the CTA's children, packed and in the reference's order (parents in chunk order, slots ascending), at
//       size - n + (children of the sub-slices before it) + ...: 8-byte stores, consecutive lanes on consecutive words
//   (7) VISIBILITY: the next round's slices must see every CTA's children, so a second exchange follows: every CTA
//       raises an epoch-tagged "stored" flag after a release fence and waits for all of them (acquire fence after).
//       It is skipped when the next round's exit tests already end the launch (the kernel boundary orders them).
// Every spin loop is guarded by SpinGuard: a stuck exchange ends the launch with RND_EXIT_ABORT (TSB_ECUDA on the
// host), never a hung GPU.
//
// One launch serves up to PFR_MAX_POOLS INDEPENDENT pools (grid (G, pools), PfRoundsMultiParams): the CTAs with
// blockIdx.y = i run pool i's rounds on pool i's arena, tables, exchange slots, state record and incumbent, and never
// wait on another pool; each pool leaves on its own exit.  With several pools every SM hosts two CTAs (pfr_tiers.h),
// so one pool's L2 round trips (count exchange, store exchange) are filled with another pool's bound work.  On an H100
// (tools/pfsp_multi_pool.py, DESIGN §4.2) the shared launch beat the same pools run one after the other at every K and
// M measured: 1.2-2.5x per pool-round, and two pools at M = 50 000 took 11.5-12.9 us per pool-round against 16.9-18.8
// for the two-kernel rounds tsb_pfsp_pool_run takes there.
#pragma once
#include "nq_rounds_ll.cuh"  // SpinGuard, RoundsState, RND_EXIT_*
#include "pfr_tiers.h"
#include "pfsp_expand.cuh"

namespace tsb {

constexpr int PFR_TILES = 3;  // tiles of 128 parents per CTA and round
static_assert(PFR_TILES * PF_TILE == PFR_SLICE, "pfr_tiers.h");

// largest M for which tsb_pfsp_pool_run takes this kernel.  On an H100 (ta014, lb1 and lb1_d, DESIGN §5) it beats the
// loop of two-kernel rounds by 1.8x at M = 300 and 1.2x at M = 20 000, and loses at M = 50 000 (18.2 against 16.4 us per
// round: a round's bound work, stores and store exchange grow with the slice, while the step loop's launch and host
// costs do not)
constexpr int PFR_MAX_M = 20000;

enum { PFR_EXIT_IMPROVED = RND_EXIT_RELAUNCH + 1 };  // (the other exit codes are nq_rounds_ll.cuh's RND_EXIT_*)

struct PfRoundsSync {
  unsigned long long slot[2 * PFR_MAX_CTAS][2];  // count slots, one per sub-slice:
                                                 // {epoch << 32 | leaves << 16 | children, epoch << 32 | leaf min}
  unsigned stored[PFR_MAX_CTAS];             // epoch of the last round whose children the CTA has stored
  unsigned abort;
};
struct PfRoundsParams {
  uint8_t* arena;                 // the pool: records [0, size0), all stored before the launch
  const PfspLb1Tables* tables;
  long long cap;                  // records the arena holds
  long long size0;
  long long max_rounds;
  unsigned epoch0;                // last epoch used so far (epochs never repeat on a handle)
  int m, M;
  int best;                       // incumbent, int32-clamped
  int prof;
  PfRoundsSync* sync;
  RoundsState* state;             // out: pool size, last epoch, exit code, counters of the committed rounds
};
struct PfRoundsMultiParams {
  PfRoundsParams pool[PFR_MAX_POOLS];  // pool blockIdx.y
};
// TSB200_ROUNDS_PROF phases (CTA 0 of each pool, thread 0 cycles)
enum { PFR_PROF_LOAD = 0, PFR_PROF_BOUND, PFR_PROF_PUBLISH, PFR_PROF_GATHER, PFR_PROF_STORE, PFR_PROF_BARRIER, PFR_PROF_N };
static_assert(PFR_PROF_N <= 12, "RoundsState::prof");

struct PfRoundsSmem {
  Lb1Smem core;                           // core.tiles.buf[0..2]: the CTA's slice (contiguous, PFR_SLICE records)
  uint32_t cmask[PFR_SLICE];              // child mask of every record of the slice
  uint16_t item[PFR_SLICE * PF_MAXJ];     // the slice's children: (record << 5) | slot, in child order
  int warp_tot[4];
  int red[4][4];                          // children of sub-slice 0, of sub-slice 1, leaves, leaf minimum per warp
  long long before[2];                    // gather: children of the sub-slices before each of this CTA's two
  long long all_children, all_leaves;
  int leaf_min;
  int ok;
  long long prof[PFR_PROF_N], prof_t;
};
static_assert(sizeof(RingSmem<PF_TILE * PF_REC>::buf) == PFR_SLICE * PF_REC, "the slice fills the tile ring");
static_assert((PFR_SLICE << 5) <= 0x10000, "item fits 16 bits");

__device__ __forceinline__ void ld_relaxed_v2(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_u32(unsigned* p, unsigned v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// (two CTAs per SM: one of each of two pools; PfRoundsSmem fits twice)
template <int KIND, int M, bool SIMD>
__global__ void __launch_bounds__(PF_THREADS, 2) pfsp_rounds_kernel(const __grid_constant__ PfRoundsMultiParams mprm) {
  const PfRoundsParams& prm = mprm.pool[blockIdx.y];
  extern __shared__ __align__(128) uint8_t smem_raw[];
  PfRoundsSmem& sm = *reinterpret_cast<PfRoundsSmem*>(smem_raw);
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int k = blockIdx.x, G = gridDim.x;
  PfRoundsSync* const sy = prm.sync;
  uint8_t* const slice = sm.core.tiles.buf[0];
  const bool prof = prm.prof != 0 && k == 0 && t == 0;
#define TSB_PFR_PROF(i)                 \
  if (prof) {                           \
    const long long now = clock64();    \
    sm.prof[i] += now - sm.prof_t;      \
    sm.prof_t = now;                    \
  }
  if (prof) {
    for (int i = 0; i < PFR_PROF_N; i++) sm.prof[i] = 0;
    sm.prof_t = clock64();
  }
  stage_blob(&sm.core.tab, prm.tables, sizeof(PfspLb1Tables), &sm.core.tab_bar);
  const int jobs = sm.core.tab.jobs, best = prm.best;

  // the pool state, the same in every thread of every CTA
  long long size = prm.size0;
  unsigned epoch = prm.epoch0;
  unsigned long long rounds = 0, tot_parents = 0, tot_children = 0, tot_solutions = 0;
  const auto exit_before = [&]() {  // (1)
    if (size < prm.m) return static_cast<int>(RND_EXIT_DONE);
    if (static_cast<long long>(rounds) >= prm.max_rounds) return static_cast<int>(RND_EXIT_PAUSE);
    const long long n = size < prm.M ? size : prm.M;
    if (size - n + n * jobs > prm.cap) return static_cast<int>(RND_EXIT_SPACE);
    return -1;
  };
  int exit_code = exit_before();
  while (exit_code < 0) {
    ++epoch;
    const long long n = size < prm.M ? size : prm.M, s0 = size - n;
    // my two sub-slices, concatenated in shared memory (n <= PFR_SLICE * G and k < G <= 256: the products fit 32 bits)
    const unsigned n32 = static_cast<unsigned>(n), uk = static_cast<unsigned>(k), uG2 = 2u * static_cast<unsigned>(G);
    const int a0 = static_cast<int>(n32 * uk / uG2), len0 = static_cast<int>(n32 * (uk + 1u) / uG2) - a0;
    const int a1 = static_cast<int>(n32 * (uG2 - 1u - uk) / uG2), len1 = static_cast<int>(n32 * (uG2 - uk) / uG2) - a1;
    const int len = len0 + len1;

    // ---- (2) my slice -> shared memory
    {
      const int2* src0 = reinterpret_cast<const int2*>(prm.arena + (s0 + a0) * PF_REC);
      const int2* src1 = reinterpret_cast<const int2*>(prm.arena + (s0 + a1) * PF_REC) - len0 * (PF_REC / 8);
      int2* dst = reinterpret_cast<int2*>(slice);
      for (int i = t; i < len * (PF_REC / 8); i += PF_THREADS) dst[i] = __ldcg((i < len0 * (PF_REC / 8) ? src0 : src1) + i);
    }
    __syncthreads();
    TSB_PFR_PROF(PFR_PROF_LOAD)

    // ---- (3) child masks, leaves, leaf minimum (pfsp_expand_count_lb1_kernel's epilogue)
    int my_children0 = 0, my_children1 = 0, my_leaves = 0, my_leaf_min = 0x7FFFFFFF;
    for (int j = 0; j * PF_TILE < len; j++) {
      const uint8_t* in_tile = slice + j * PF_TILE * PF_REC;
      const int hi = min(PF_TILE, len - j * PF_TILE);
      uint32_t mk = 0, live = 0;
      int leaf_lb = 0x7FFFFFFF;
      const int p = lb1_compute_tile<KIND, M, SIMD, false>(sm.core, in_tile, 0, hi,
                                                           [&](int, int limit1, int g, const int(&v)[4]) {
#pragma unroll
                                                             for (int c = 0; c < 4; c++) {
                                                               const int s = 4 * g + c;
                                                               if (s > limit1) {
                                                                 live |= 1u << s;
                                                                 if (v[c] < best) mk |= 1u << s;
                                                                 leaf_lb = min(leaf_lb, v[c]);
                                                               }
                                                             }
                                                           });
      if (live) {  // p is a valid parent with at least one slot
        const int depth = reinterpret_cast<const int32_t*>(in_tile)[22 * p];
        if (depth + 1 == jobs) {  // every child is a leaf (pfsp_gpu_chpl.chpl:283-288)
          my_leaves += __popc(live);
          mk = 0;
          my_leaf_min = min(my_leaf_min, leaf_lb);
        }
      }
      sm.cmask[j * PF_TILE + p] = mk;  // (p runs over all 128 records of the tile)
      if (j * PF_TILE + p < len0)
        my_children0 += __popc(mk);
      else
        my_children1 += __popc(mk);
    }
    // CTA totals
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      my_children0 += __shfl_xor_sync(0xFFFFFFFFu, my_children0, o);
      my_children1 += __shfl_xor_sync(0xFFFFFFFFu, my_children1, o);
      my_leaves += __shfl_xor_sync(0xFFFFFFFFu, my_leaves, o);
      my_leaf_min = min(my_leaf_min, __shfl_xor_sync(0xFFFFFFFFu, my_leaf_min, o));
    }
    if (lane == 0) {
      sm.red[0][wid] = my_children0;
      sm.red[1][wid] = my_children1;
      sm.red[2][wid] = my_leaves;
      sm.red[3][wid] = my_leaf_min;
    }
    __syncthreads();  // (also: every thread's cmask entries are written)
    const int children0 = sm.red[0][0] + sm.red[0][1] + sm.red[0][2] + sm.red[0][3];
    const int cta_children = children0 + sm.red[1][0] + sm.red[1][1] + sm.red[1][2] + sm.red[1][3];
    TSB_PFR_PROF(PFR_PROF_BOUND)

    // ---- (4) publish (the whole slice is in shared memory: the barrier above follows the loads of (2))
    if (t < 2) {  // slot k: sub-slice 0 with the CTA's leaf statistics; slot 2G-1-k: sub-slice 1
      const int leaves = t ? 0 : sm.red[2][0] + sm.red[2][1] + sm.red[2][2] + sm.red[2][3];
      const int lmin = t ? 0x7FFFFFFF : min(min(sm.red[3][0], sm.red[3][1]), min(sm.red[3][2], sm.red[3][3]));
      const unsigned long long e = static_cast<unsigned long long>(epoch) << 32;
      // (children and leaves of a slice are < PFR_SLICE * 20 < 2^16)
      asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(sy->slot[t ? 2 * G - 1 - k : k]),
                   "l"(e | static_cast<unsigned long long>(leaves) << 16 |
                       static_cast<unsigned>(t ? cta_children - children0 : children0)),
                   "l"(e | static_cast<unsigned>(lmin))
                   : "memory");
    }
    // the child list of the slice while the other CTAs publish: block scan of the child counts, tile by tile
    {
      int base = 0;
      for (int j = 0; j * PF_TILE < len; j++) {
        const int r = j * PF_TILE + t;
        const uint32_t cm = sm.cmask[r];
        const int mine = __popc(cm);
        int incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
          if (lane >= o) incl += y;
        }
        if (lane == 31) sm.warp_tot[wid] = incl;
        __syncthreads();
        int pos = base + incl - mine, total = 0;
#pragma unroll
        for (int i = 0; i < 4; i++) {
          if (i < wid) pos += sm.warp_tot[i];
          total += sm.warp_tot[i];
        }
        for (uint32_t m = cm; m; m &= m - 1) sm.item[pos++] = static_cast<uint16_t>(r << 5 | (__ffs(m) - 1));
        base += total;
        __syncthreads();  // (warp_tot is rewritten by the next tile)
      }
    }
    TSB_PFR_PROF(PFR_PROF_PUBLISH)
    // gather every slot (warp 0; every lane holds the sums at the end)
    if (wid == 0) {
      SpinGuard guard;
      bool ok = true;
      long long before0 = 0, before1 = 0, all_c = 0, all_l = 0;
      int lmin = 0x7FFFFFFF;
      const int G2 = 2 * G, k1 = G2 - 1 - k;
      for (;;) {
        unsigned long long v0[2 * PFR_MAX_CTAS / 32], v1[2 * PFR_MAX_CTAS / 32];
#pragma unroll
        for (int u = 0; u < 2 * PFR_MAX_CTAS / 32; u++)
          if (lane + 32 * u < G2) ld_relaxed_v2(sy->slot[lane + 32 * u], v0[u], v1[u]);
        bool have = true;
        before0 = before1 = all_c = all_l = 0;
        lmin = 0x7FFFFFFF;
#pragma unroll
        for (int u = 0; u < 2 * PFR_MAX_CTAS / 32; u++) {
          const int i = lane + 32 * u;
          if (i < G2) {
            have &= static_cast<unsigned>(v0[u] >> 32) == epoch && static_cast<unsigned>(v1[u] >> 32) == epoch;
            const long long c = static_cast<long long>(v0[u] & 0xFFFFu);
            all_c += c;
            if (i < k) before0 += c;
            if (i < k1) before1 += c;
            all_l += static_cast<long long>((v0[u] >> 16) & 0xFFFFu);
            lmin = min(lmin, static_cast<int>(static_cast<unsigned>(v1[u])));
          }
        }
        if (__all_sync(0xFFFFFFFFu, have)) break;
        if (__any_sync(0xFFFFFFFFu, guard.expired(&sy->abort))) {
          ok = false;
          break;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        before0 += __shfl_xor_sync(0xFFFFFFFFu, before0, o);
        before1 += __shfl_xor_sync(0xFFFFFFFFu, before1, o);
        all_c += __shfl_xor_sync(0xFFFFFFFFu, all_c, o);
        all_l += __shfl_xor_sync(0xFFFFFFFFu, all_l, o);
        lmin = min(lmin, __shfl_xor_sync(0xFFFFFFFFu, lmin, o));
      }
      if (lane == 0) {
        sm.before[0] = before0;
        sm.before[1] = before1;
        sm.all_children = all_c;
        sm.all_leaves = all_l;
        sm.leaf_min = lmin;
        sm.ok = ok;
      }
    }
    __syncthreads();
    TSB_PFR_PROF(PFR_PROF_GATHER)
    // ---- (5) uniform decisions, before any store
    if (!sm.ok) {
      exit_code = RND_EXIT_ABORT;
      break;
    }
    if (sm.leaf_min < best) {
      exit_code = PFR_EXIT_IMPROVED;
      break;
    }
    const long long round_children = sm.all_children;

    // ---- (6) the children: word w of the CTA's run is word w % 11 of child w / 11 (the first children0 children
    // are sub-slice 0's); four independent words per thread and step
    {
      constexpr int W = PF_REC / 8;
      int2* const g0 = reinterpret_cast<int2*>(prm.arena + (s0 + sm.before[0]) * PF_REC);
      int2* const g1 = reinterpret_cast<int2*>(prm.arena + (s0 + sm.before[1]) * PF_REC) - children0 * W;
      const int words = cta_children * W;
#pragma unroll 4
      for (int w = t; w < words; w += PF_THREADS) {
        const int c = w / W, i = w - c * W;
        const int item = sm.item[c];
        const int32_t* par = reinterpret_cast<const int32_t*>(slice + (item >> 5) * PF_REC);
        const int jd = par[0] + 2, jk = (item & 31) + 2;  // int32 index of prmu[depth] and of prmu[slot]
        int x = par[2 * i], y = par[2 * i + 1];
        if (i == 0) {  // depth + 1, limit1 + 1
          ++x;
          ++y;
        }
        if (2 * i == jd) x = par[jk]; else if (2 * i == jk) x = par[jd];
        if (2 * i + 1 == jd) y = par[jk]; else if (2 * i + 1 == jk) y = par[jd];
        (c < children0 ? g0 : g1)[w] = make_int2(x, y);
      }
    }
    TSB_PFR_PROF(PFR_PROF_STORE)
    // ---- the pool after the round
    size = s0 + round_children;
    ++rounds;
    tot_parents += static_cast<unsigned long long>(n);
    tot_children += static_cast<unsigned long long>(round_children);
    tot_solutions += static_cast<unsigned long long>(sm.all_leaves);
    exit_code = exit_before();
    if (exit_code >= 0) break;
    // ---- (7) every CTA's children stored before any CTA reads the next chunk
    __syncthreads();  // (also: nobody still reads sm.before / sm.item of this round)
    if (wid == 0) {
      if (lane == 0) {
        __threadfence();
        st_relaxed_u32(&sy->stored[k], epoch);
      }
      SpinGuard guard;
      bool ok = true;
      for (;;) {
        bool have = true;
#pragma unroll
        for (int u = 0; u < PFR_MAX_CTAS / 32; u++)
          if (lane + 32 * u < G) have &= ld_relaxed_u32(&sy->stored[lane + 32 * u]) == epoch;
        if (__all_sync(0xFFFFFFFFu, have)) break;
        if (__any_sync(0xFFFFFFFFu, guard.expired(&sy->abort))) {
          ok = false;
          break;
        }
      }
      __threadfence();
      if (lane == 0) sm.ok = ok;
    }
    __syncthreads();
    TSB_PFR_PROF(PFR_PROF_BARRIER)
    if (!sm.ok) {
      exit_code = RND_EXIT_ABORT;
      break;
    }
  }
#undef TSB_PFR_PROF
  if (k == 0 && t == 0) {
    RoundsState* st = prm.state;
    st->size = size;
    st->epoch = epoch;
    st->rounds = rounds;
    st->parents = tot_parents;
    st->children = tot_children;
    st->solutions = tot_solutions;
    if (prm.prof)
      for (int i = 0; i < PFR_PROF_N; i++) st->prof[i] = sm.prof[i];
    __threadfence_system();
    *reinterpret_cast<volatile int*>(&st->exit_code) = exit_code;
  }
}

}  // namespace tsb

// pfsp_wide_rounds.cuh — the persistent multi-round PFSP kernel for 208-byte tsb_pfsp_node50 records (the reference
// built with MAX_JOBS = 50, ta031..ta060), lb1 / lb1_d, sm_90a (H100).
//
// The contract of pfsp_rounds_kernel (pfsp_rounds.cuh): the whole offload loop of a 50-job device pool in one
// cooperative launch instead of the two kernels of pfsp_wide_expand.cuh and a host wait per round; the pool is one
// contiguous stack [0, size) in the arena while the kernel runs; grid (G, pools), blockIdx.y = the pool; the same exit
// codes (DONE, PAUSE exactly at max_rounds, SPACE, PFR_EXIT_IMPROVED decided before any store, the round then not
// committed) and the same two epoch-tagged exchanges per round, every spin loop under SpinGuard.  A round:
//   (1) exit tests; the chunk is the top n = min(size, M) records, cut into 2G sub-slices: CTA k takes number k from
//       the bottom and number k from the top (the pairing of pfsp_rounds.cuh)
//   (2) the CTA's slice (at most PFR_SLICE = 384 records, 79 872 bytes) -> shared memory, 16-byte L2 loads
//   (3) one thread per parent: pw_parent_bounds (pfsp_wide.cuh, the bound code of the evaluator and of the count
//       kernel) with each bound folded at once into the parent's 64-bit child mask, leaf count and leaf minimum (no
//       bound array: 384 x 50 bounds would not leave room for two CTAs per SM)
//   (4) count exchange: publish {children, leaves, leaf minimum} of both sub-slices, block scan of the child counts,
//       gather every slot
//   (5) IMPROVED (uniform): the chunk's leaf minimum is below `best`: nothing is stored, the host redoes the round
//   (6) the children, in the reference's order (parents in chunk order, slots ascending), stored in place, one tile of
//       PFW_TILE parents at a time: the tile's child list (parent, slot) in shared memory, then whole 16-byte words,
//       consecutive threads on consecutive words (208 = 13 x 16)
//   (7) store exchange: every CTA's children are visible before any CTA reads the next chunk (skipped when the next
//       round's exit tests end the launch)
// Shared memory: 98 KB per CTA (slice 79 872, lb1 tables 5 232, one tile's child list 12 800; each parent's child mask
// stays in its thread's registers), so two CTAs fit on an SM: the capacities of pfr_tiers.h hold unchanged (50 688
// parents per pool for K <= 2 on 132 SMs).
#pragma once
#include "pfsp_rounds.cuh"      // PfRoundsSync, PFR_EXIT_IMPROVED, PFR_PROF_*, the relaxed loads and stores
#include "pfsp_wide_expand.cuh" // PW_WORDS

namespace tsb {

constexpr int PFW_THREADS = PFR_SLICE;  // one thread per parent of the slice
constexpr int PFW_WARPS = PFW_THREADS / 32;
constexpr int PFW_TILE = 128;           // parents whose children are listed and stored at once
constexpr int PFW_TILES = PFR_SLICE / PFW_TILE;
static_assert(PFW_TILES * PFW_TILE == PFR_SLICE && PFW_TILE % 32 == 0, "a tile is whole warps");
static_assert((PFW_TILE << 6) <= 0x10000, "item fits 16 bits");

struct PfWideRoundsParams {
  uint8_t* arena;                 // the pool: records [0, size0), all stored before the launch
  const PfspWideTables* tables;
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
struct PfWideRoundsMultiParams {
  PfWideRoundsParams pool[PFR_MAX_POOLS];  // pool blockIdx.y
};

struct PfWideRoundsSmem {
  alignas(16) int32_t slice[PFR_SLICE * (PW_REC / 4)];  // the CTA's two sub-slices, concatenated
  alignas(16) uint8_t tab[offsetof(PfspWideTables, jp)];  // PfspWideTables without the Johnson words (lb2 only)
  uint16_t item[PFW_TILE * PW_MAXJ];  // one tile's children: (parent in the tile << 6) | slot, in child order
  int warp_tot[PFW_WARPS];            // children of each warp's parents
  int red[3][PFW_WARPS];              // children of sub-slice 0, leaves, leaf minimum per warp
  long long before[2];                // gather: children of the sub-slices before each of this CTA's two
  long long all_children, all_leaves;
  int leaf_min;
  int ok;
  long long prof[PFR_PROF_N], prof_t;
};

// two CTAs per SM, of one pool or of two
template <int KIND, int M>
__global__ void __launch_bounds__(PFW_THREADS, 2) pfsp_wide_rounds_kernel(const __grid_constant__ PfWideRoundsMultiParams mprm) {
  static_assert(KIND == 0 || KIND == 1, "lb1_d and lb1 only");
  const PfWideRoundsParams& prm = mprm.pool[blockIdx.y];
  extern __shared__ __align__(128) uint8_t smem_raw[];
  PfWideRoundsSmem& sm = *reinterpret_cast<PfWideRoundsSmem*>(smem_raw);
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int k = blockIdx.x, G = gridDim.x;
  PfRoundsSync* const sy = prm.sync;
  const PfspWideTables& tab = *reinterpret_cast<const PfspWideTables*>(sm.tab);
  const bool prof = prm.prof != 0 && k == 0 && t == 0;
#define TSB_PFW_PROF(i)                 \
  if (prof) {                           \
    const long long now = clock64();    \
    sm.prof[i] += now - sm.prof_t;      \
    sm.prof_t = now;                    \
  }
  if (prof) {
    for (int i = 0; i < PFR_PROF_N; i++) sm.prof[i] = 0;
    sm.prof_t = clock64();
  }
  pw_stage_tables<KIND>(reinterpret_cast<PfspWideTables*>(sm.tab), prm.tables);
  __syncthreads();
  const int jobs = tab.jobs, best = prm.best;

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
    // my two sub-slices (n <= PFR_SLICE * G and k < G <= 256: the products fit 32 bits)
    const unsigned n32 = static_cast<unsigned>(n), uk = static_cast<unsigned>(k), uG2 = 2u * static_cast<unsigned>(G);
    const int a0 = static_cast<int>(n32 * uk / uG2), len0 = static_cast<int>(n32 * (uk + 1u) / uG2) - a0;
    const int a1 = static_cast<int>(n32 * (uG2 - 1u - uk) / uG2), len1 = static_cast<int>(n32 * (uG2 - uk) / uG2) - a1;
    const int len = len0 + len1;

    // ---- (2) my slice -> shared memory
    {
      const uint4* src0 = reinterpret_cast<const uint4*>(prm.arena + (s0 + a0) * PW_REC);
      const uint4* src1 = reinterpret_cast<const uint4*>(prm.arena + (s0 + a1) * PW_REC) - len0 * PW_WORDS;
      uint4* dst = reinterpret_cast<uint4*>(sm.slice);
      for (int i = t; i < len * PW_WORDS; i += PFW_THREADS) dst[i] = __ldcg((i < len0 * PW_WORDS ? src0 : src1) + i);
    }
    __syncthreads();
    TSB_PFW_PROF(PFR_PROF_LOAD)

    // ---- (3) my parent's child mask, leaves, leaf minimum (pfsp_wide_expand_count_kernel's epilogue)
    unsigned long long mk = 0;
    int leaves = 0, leaf_min = 0x7FFFFFFF;
    if (t < len) {
      const int32_t* node = sm.slice + t * (PW_REC / 4);
      int lmin = 0x7FFFFFFF;
      pw_parent_bounds<KIND, M>(tab, node, nullptr, best, [&](int s, int lb) {
        if (lb < best) mk |= 1ull << s;
        lmin = min(lmin, lb);
      });
      if (node[0] + 1 == jobs) {  // every child is a leaf (pfsp_gpu_chpl.chpl:283-288)
        leaves = jobs - 1 - min(max(node[1], -1), jobs - 1);
        leaf_min = lmin;
        mk = 0;
      }
    }
    const int mine = __popcll(mk);
    // block scan of the child counts (my parent's first child in the CTA's run) and the CTA totals
    int incl = mine, c0 = t < len0 ? mine : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= o) incl += y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      c0 += __shfl_xor_sync(0xFFFFFFFFu, c0, o);
      leaves += __shfl_xor_sync(0xFFFFFFFFu, leaves, o);
      leaf_min = min(leaf_min, __shfl_xor_sync(0xFFFFFFFFu, leaf_min, o));
    }
    if (lane == 31) sm.warp_tot[wid] = incl;
    if (lane == 0) {
      sm.red[0][wid] = c0;
      sm.red[1][wid] = leaves;
      sm.red[2][wid] = leaf_min;
    }
    __syncthreads();
    int pos = incl - mine, children0 = 0, cta_children = 0, cta_leaves = 0, cta_leaf_min = 0x7FFFFFFF;
#pragma unroll
    for (int i = 0; i < PFW_WARPS; i++) {
      if (i < wid) pos += sm.warp_tot[i];
      cta_children += sm.warp_tot[i];
      children0 += sm.red[0][i];
      cta_leaves += sm.red[1][i];
      cta_leaf_min = min(cta_leaf_min, sm.red[2][i]);
    }
    TSB_PFW_PROF(PFR_PROF_BOUND)

    // ---- (4) publish (the whole slice is in shared memory: the barrier above follows the loads of (2)): slot k:
    // sub-slice 0 with the CTA's leaf statistics; slot 2G-1-k: sub-slice 1
    if (t < 2) {
      const unsigned long long e = static_cast<unsigned long long>(epoch) << 32;
      // (children and leaves of a slice are < PFR_SLICE * 50 < 2^16)
      asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(sy->slot[t ? 2 * G - 1 - k : k]),
                   "l"(e | static_cast<unsigned long long>(t ? 0 : cta_leaves) << 16 |
                       static_cast<unsigned>(t ? cta_children - children0 : children0)),
                   "l"(e | static_cast<unsigned>(t ? 0x7FFFFFFF : cta_leaf_min))
                   : "memory");
    }
    TSB_PFW_PROF(PFR_PROF_PUBLISH)
    // gather every slot (warp 0; every lane holds the sums at the end)
    if (wid == 0) {
      SpinGuard guard;
      bool ok = true;
      long long before0 = 0, before1 = 0, all_c = 0, all_l = 0;
      int lmin = 0x7FFFFFFF;
      const int G2 = 2 * G, k1 = G2 - 1 - k;
      for (;;) {
        bool have = true;
        before0 = before1 = all_c = all_l = 0;
        lmin = 0x7FFFFFFF;
        // (each slot taken as it is loaded: the 20-job kernel's arrays of all 16 slots per lane do not fit the 80
        // registers of two 384-thread CTAs per SM)
#pragma unroll 4
        for (int u = 0; u < 2 * PFR_MAX_CTAS / 32; u++) {
          const int i = lane + 32 * u;
          if (i < G2) {
            unsigned long long v0, v1;
            ld_relaxed_v2(sy->slot[i], v0, v1);
            have &= static_cast<unsigned>(v0 >> 32) == epoch && static_cast<unsigned>(v1 >> 32) == epoch;
            const long long c = static_cast<long long>(v0 & 0xFFFFu);
            all_c += c;
            if (i < k) before0 += c;
            if (i < k1) before1 += c;
            all_l += static_cast<long long>((v0 >> 16) & 0xFFFFu);
            lmin = min(lmin, static_cast<int>(static_cast<unsigned>(v1)));
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
    TSB_PFW_PROF(PFR_PROF_GATHER)
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

    // ---- (6) the children, tile by tile: child c of the CTA's run (the first children0 are sub-slice 0's) is word
    // range [13 c, 13 c + 13) of g0, or of g1 for sub-slice 1
    {
      int4* const g0 = reinterpret_cast<int4*>(prm.arena + (s0 + sm.before[0]) * PW_REC);
      int4* const g1 = reinterpret_cast<int4*>(prm.arena + (s0 + sm.before[1]) * PW_REC) - children0 * PW_WORDS;
      int tile_base = 0;
#pragma unroll 1
      for (int j = 0; j < PFW_TILES; j++) {
        int tile_children = 0;
#pragma unroll
        for (int i = 0; i < PFW_TILE / 32; i++) tile_children += sm.warp_tot[j * (PFW_TILE / 32) + i];
        if (tile_children == 0) continue;  // (uniform)
        if (t / PFW_TILE == j) {
          int p = pos - tile_base;
          for (unsigned long long m = mk; m; m &= m - 1)
            sm.item[p++] = static_cast<uint16_t>((t - j * PFW_TILE) << 6 | (__ffsll(m) - 1));
        }
        __syncthreads();
        for (int w = t; w < tile_children * PW_WORDS; w += PFW_THREADS) {
          const int c = w / PW_WORDS, i = w - c * PW_WORDS;
          const int item = sm.item[c];
          const int32_t* src = sm.slice + (j * PFW_TILE + (item >> 6)) * (PW_REC / 4);
          const int s = item & 63, depth = src[0];
          const int4 v = reinterpret_cast<const int4*>(src)[i];
          int e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int q = 0; q < 4; q++) {  // int 4i + q of the record: depth, limit1, prmu[0..50)
            const int x = 4 * i + q;
            if (x == 0) e[q] = depth + 1;
            else if (x == 1) e[q] = src[1] + 1;
            else if (x == 2 + depth) e[q] = src[2 + s];  // child.prmu[depth] <=> child.prmu[s]
            else if (x == 2 + s) e[q] = src[2 + depth];
          }
          const int cc = tile_base + c;
          (cc < children0 ? g0 : g1)[cc * PW_WORDS + i] = make_int4(e[0], e[1], e[2], e[3]);
        }
        tile_base += tile_children;
        __syncthreads();  // (the next tile rewrites the child list)
      }
    }
    TSB_PFW_PROF(PFR_PROF_STORE)
    // ---- the pool after the round
    size = s0 + round_children;
    ++rounds;
    tot_parents += static_cast<unsigned long long>(n);
    tot_children += static_cast<unsigned long long>(round_children);
    tot_solutions += static_cast<unsigned long long>(sm.all_leaves);
    exit_code = exit_before();
    if (exit_code >= 0) break;
    // ---- (7) every CTA's children stored before any CTA reads the next chunk
    __syncthreads();  // (also: nobody still reads sm.before / sm.warp_tot / sm.all_leaves of this round)
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
    TSB_PFW_PROF(PFR_PROF_BARRIER)
    if (!sm.ok) {
      exit_code = RND_EXIT_ABORT;
      break;
    }
  }
#undef TSB_PFW_PROF
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

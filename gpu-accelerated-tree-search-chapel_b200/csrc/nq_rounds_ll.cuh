// nq_rounds_ll.cuh — the persistent multi-round N-Queens kernel without fences on its critical path.
//
// One round of the reference's step 2 (nqueens_gpu_chpl.chpl:197-215) is: popBackBulk(m, M) = the newest
// n = min(size, M) nodes of the pool (nothing if size < m, lib/commons/Pool.chpl:50-59), evaluate_gpu on them,
// generate_children pushing the surviving children back, in order.  Round i+1 pops what round i pushed, so the rounds
// are a latency chain; at the reference's default --M 50000 two launches and a host poll per round would be the cost.
// This kernel runs the whole loop in one cooperative launch: every CTA tracks the (tiny) pool state redundantly — a
// deterministic function of the per-round totals, which every CTA learns anyway — so nothing is broadcast.  Inside a
// CTA, eight worker warps move and build the nodes and a ninth, the EXCHANGE warp, owns the count exchange and the
// pool state (the round is described above nq_rounds_ll_kernel).
//
// An earlier version ordered round r+1 after round r with a release fence (MEMBAR.ALL.GPU, thousands of cycles under
// load) and a "done" flag exchange among all CTAs, on top of the exchange that gathers the child counts: most of its
// round was spent waiting on them (rounds_sync_bench_kernel at the end of this file measures that floor).  It was
// removed in favour of this kernel.  Here the pool lives, while the kernel runs, in a SELF-VALIDATING format
// (the "LL" idea of NCCL's low-latency protocol):
//
//   fat node = 4 x 8-byte words; word i = data32[i] | x16[i] << 32 | tag << 48   (32 B per node = one sector,
//   32-byte aligned), read and written as two 16-byte pieces (words 0-1 and 2-3)
//   data32[0..3] = the node packed in 125 bits (any N <= 24: every board value is below 32):
//     board[i] in bits 5 (i % 6) .. +4 of data32[i / 6]            (six values per word)
//     depth in the 2-bit tails (bits 30..31) of data32[0], [1], [2]: bits 0-1, 2-3 and 4 of the depth
//     21-byte records (N <= 20): data32[3] holds board[18], [19] in bits 0..9, then bits 10..29: the node's child mask
//     (slot k set <=> k >= depth and board[k] is not attacked: evaluate_gpu's label for slot k,
//     nqueens_gpu_chpl.chpl:97-123), bit 30: leaf (depth == N)
//     25-byte records (a wide handle, N <= 24): data32[3] holds board[18..23] in bits 0..29; neither the child mask
//     nor the leaf flag is stored: a leaf is depth == N, and the child mask is evaluated when the node is read as a
//     parent, from its board and its diagonal masks (ll_child_mask: a few slots, most parents lie at depth N-4..N-3)
//   x16[0..3] = the node's diagonal masks, the values its next row attacks (N bits each):
//     ld (rising diagonals) = x16[0] | x16[1] << 16, in piece 0; rd (falling diagonals) = x16[2] | x16[3] << 16, in piece 1
//   tag = the 16-bit tag of the epoch the word was stored in (ll_tag; 0: no round's tag, see below)
//   A child's masks follow from its parent's in O(1) and (21-byte records) its child mask is evaluated from them when it
//   is built (ll_build_child), so a round reads its parents' masks instead of recomputing them from the placed prefix.
//   (An earlier version stored the masks in a side word next to each 21-byte node: 64 bytes per node, twice the poll
//   loads and store pieces of a round.)
//
// Every 8-byte word is written by one store (an element of a st.v2.u64) and is therefore seen whole or not at all;
// a reader that expects the children of round r polls the words of its slice until all four carry r's tag.  No
// fence, no "done" flags: the data is its own flag, and a round costs ONE flag exchange (the child counts) plus one
// store -> L2 -> poll hop for the nodes.
//
// Tags are 16 bits, so they repeat, and a stale word must never carry the tag a reader expects at its position.
// Epochs count rounds (32 bits, never repeating; the count slots of LlSync carry them whole) and tag(e) = e mod 65535
// + 1 (ll_tag), so tag 0 belongs to no epoch and epochs less than 65535 apart have different tags.  Per pool the host
// keeps the epoch C of the last CLEAR, which sets the tag of every word of the arena to 0 (data kept; a new arena is
// zeroed, and the import from the plain arena stores tag 0), and a launch uses epochs up to C + LL_TAG_SPAN at most
// (LlParams::epoch_last: the kernel leaves with RND_EXIT_RELAUNCH there; the host clears before a launch that would
// have too few epochs left, ll_tag_window).  So every word of the arena carries tag 0 or the tag of an epoch e' with
// C < e' < e for any live epoch e <= C + LL_TAG_SPAN: 0 < e - e' < 65535, the tags differ, and tag 0 is no live
// round's.  A clear re-tags only the positions below the highest pool size reached since the previous clear
// (RoundsState::size_hi: every store of a launch lies below it), about once per 65 000 rounds.
//
// Nodes that are NOT children of the previous round (the chunk reaches below the newest layer when a round produced
// fewer than M children) carry the epoch of the round that stored them.  Every CTA keeps the LAYER STACK of the pool
// — (first position, epoch) of every round's children that are still in the pool, a deterministic function of the
// round totals like the rest of the pool state — and validates every piece against the epoch of the layer its
// position lies in.  Nodes that were in the pool when the kernel was launched form one trusted layer (a kernel
// boundary orders them).  (A first version fenced old rounds with a side warp and checked per-CTA fence flags before
// reading old nodes: that check sat on the critical path of every round that reaches below the newest layer.)
//
// Alternatives tried for the one remaining exchange (all CTAs polling the 2 G count words): a dedicated aggregator
// CTA that scans the counts and writes every worker its own result line (two contention-free hops, no gain),
// per-reader rows that only their owner polls (no gain), CTAs of 512 threads (slower scan), fewer CTAs (cheaper
// exchange, more work per CTA: the default uses 7/8 of the SMs), a sentinel poll (one lane per warp watches one piece
// and the full sweeps start when it has arrived: the extra hop costs more than the poll traffic it saves).  Taking the
// exchange out of the round altogether, with the next round's counts published next to the children, measured 1.65x
// slower (DESIGN §5): the in-place stores then need their own "every slice read" wait, and the build is no longer hidden.
// What did pay: the same 256 worker threads plus one exchange warp per CTA.  Warp 0 used to start the gather only after
// its share of the build, and all eight warps ran the round's bookkeeping and the next round's set-up after their
// stores, behind two CTA barriers; the exchange warp gathers while the workers build and does the bookkeeping before
// the handoff, so the workers go from their stores straight into the next poll (6 % faster, DESIGN §5).
//
// The plain arena (21- or 25-byte records) is converted
// to and from the fat arena by nq_fat_import / nq_fat_export (whole pool, only when the host needs the plain form:
// drain, steal, pool_step, arena growth).
//
// One launch serves up to LL_MAX_POOLS INDEPENDENT pools (grid (G, pools), LlMultiParams): even so a pool's round stays
// a chain of L2 round trips with little work in between, and nothing inside one pool can fill the waits — another
// pool's CTA on the same SM can: on the N = 17 search at M = 50000 three or four pools per launch (two pools per SM in
// all, 768 parents per CTA) take little more than half the time of one pool.  Four pools run as grid (G, 2) of CTAs
// that each hold two pools' CTAs as halves (HALVES, above nq_rounds_ll_kernel).  Pools of 25-byte records run one per
// launch (nq_rounds_ll_wide_kernel).
//
// A spin loop that waits longer than ~2 s raises a global abort flag and every CTA leaves (exit code ABORT): a logic
// error must never hang the GPU.
#pragma once
#include "ll_tiers.h"
#include "nq_kernel.cuh"

namespace tsb {

constexpr int LL_T = 256;                    // worker threads per CTA (plus the exchange warp)
// parents per worker thread (PPT): 2 with one or two pools per launch (7/8 of the SMs / all SMs per pool), 3 with three or four
// (SMs / 2 CTAs per pool: a round's count exchange among half the CTAs costs about half, tools/flag_exchange.py, and
// every CTA brings 1.5x the work to hide it behind)
__host__ __device__ constexpr int ll_slice(int ppt) { return LL_T * ppt; }          // parents per CTA per round
static_assert(ll_slice(2) == LL_SLICE2 && ll_slice(3) == LL_SLICE3, "ll_tiers.h");

enum { RND_EXIT_DONE = 0, RND_EXIT_PAUSE = 1, RND_EXIT_SPACE = 2, RND_EXIT_ABORT = 3, RND_EXIT_RELAUNCH = 4 };
// in / out record of a launch (pinned + mapped host memory)
struct RoundsState {
  long long size;                 // nodes in the pool: positions [0, size)
  unsigned epoch;                 // last epoch used
  int exit_code;
  unsigned long long rounds, parents, children, solutions;  // of this launch
  long long prof[12];  // (prm.prof) cycles CTA 0 spent per phase (the LL_PROF_* indices of nq_rounds_ll_kernel)
  long long size_hi;   // (nq_rounds_ll_kernel) the largest pool size of the launch: every position it stored lies below
  // (nq_rounds_ll_kernel, prm.prof) %globaltimer (ns) read by CTA 0's exchange warp when the pool starts and when it
  // leaves the launch (a launch ends when its last pool leaves), and where each CTA k of the pool ran: %smid and the
  // low 32 bits of %globaltimer at its start
  unsigned long long t_start, t_exit;
  unsigned cta_sm[LL_MAX_SMS], cta_t0[LL_MAX_SMS];
  // (prm.prof) per CTA k: parents of its sub-slices that had children, and rounds whose children took more than one
  // staging window (LL_CAP)
  unsigned cta_fertile[LL_MAX_SMS], cta_wide[LL_MAX_SMS];
};
__device__ __forceinline__ unsigned long long ll_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ unsigned ll_smid() {
  unsigned s;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
  return s;
}

__device__ __forceinline__ void st_relaxed_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// Every CTA needs every other CTA's flag, so the polling is done by ONE warp per CTA with coalesced 16-byte loads: one
// thread per slot spinning on its own flag put ~22 000 loads per sweep on a handful of L2 lines and made rounds
// several times slower.
struct SpinGuard {  // watchdog of a spin loop: ~2 s, or another CTA's abort
  unsigned spins = 0;
  long long t0 = 0;
  __device__ __forceinline__ bool expired(unsigned* abort_flag) {
    if ((++spins & 0xFFu) != 0) return false;
    if (*reinterpret_cast<volatile unsigned*>(abort_flag)) return true;
    const long long now = clock64();
    if (t0 == 0) t0 = now;
    if (now - t0 > 4000000000LL) {
      *reinterpret_cast<volatile unsigned*>(abort_flag) = 1u;
      return true;
    }
    return false;
  }
};
// children per window of the staging buffer (a CTA's share of a round averages ~0.8 children per parent; a dense
// share takes several windows)
constexpr int LL_CAP = 2048;
constexpr int LL_WORDS = 4;                  // 8-byte words per fat node
constexpr int LL_LAYERS = 1024;              // layers of the pool a CTA tracks (more: the kernel leaves and is relaunched)
constexpr unsigned LL_TRUSTED = 0u;          // layer tag of the nodes that were in the pool at launch (no round's tag)
// the 16-bit tag of epoch e: 1 .. 65535 (see above; LL_TAG_SPAN and the host's clear decision: ll_tiers.h)
__device__ __forceinline__ unsigned ll_tag(unsigned e) { return e % LL_TAG_SPAN + 1u; }

struct alignas(32) FatNode {
  unsigned long long w[LL_WORDS];
};
// a 16-byte piece of a fat node from two data words and the piece's diagonal mask (ld for piece 0, rd for piece 1)
// and tag: x16 = the mask's low half in the first word, its high half in the second
__device__ __forceinline__ void ll_piece(uint32_t d0, uint32_t d1, uint32_t mask, uint32_t tag, unsigned long long& a,
                                         unsigned long long& b) {
  a = static_cast<unsigned long long>(__byte_perm(mask, tag, 0x5410)) << 32 | d0;
  b = static_cast<unsigned long long>(__byte_perm(mask, tag, 0x5432)) << 32 | d1;
}
// the packed node (data32[0..3], see above)
constexpr int LL_CM_SHIFT = 10;          // (21-byte records) child mask: data32[3] bits 10..29
constexpr uint32_t LL_LEAF = 1u << 30;   // (21-byte records) leaf flag: data32[3] bit 30
__host__ __device__ constexpr int ll_fw(int i) { return i / 6; }        // data word of board[i]
__host__ __device__ constexpr int ll_fs(int i) { return 5 * (i % 6); }  // its first bit
__device__ __forceinline__ uint32_t ll_depth(uint32_t d0, uint32_t d1, uint32_t d2) {
  return d0 >> 30 | (d1 >> 30) << 2 | (d2 >> 30) << 4;
}
// data32[0..2] with their depth tails replaced by those of `depth`
__device__ __forceinline__ void ll_set_depth(uint32_t (&d)[4], uint32_t depth) {
  d[0] = (d[0] & 0x3FFFFFFFu) | (depth & 3u) << 30;
  d[1] = (d[1] & 0x3FFFFFFFu) | (depth >> 2 & 3u) << 30;
  d[2] = (d[2] & 0x3FFFFFFFu) | (depth >> 4) << 30;
}
struct LlSync {
  unsigned long long slot[2][2 * LL_MAX_SMS];  // by round parity, one per SUB-slice: epoch << 32 | leaves << 20 | children
  unsigned abort;
};
constexpr int LL_MAX_POOLS = 4;  // independent pools one launch can serve (blockIdx.y)
struct LlParams {
  FatNode* fat;
  long long cap;    // nodes the fat arena holds
  long long size0;  // nodes in the pool at launch: positions [0, size0), all stored before the launch
  unsigned epoch0;      // last epoch used so far (the previous launch's last round)
  unsigned epoch_last;  // the last epoch this launch may use (ll_tag_window)
  int m, M;
  long long max_rounds;
  int prof;
  LlSync* sync;
  RoundsState* state;
};
// Several INDEPENDENT pools in one cooperative launch: grid (G, pools), the CTAs of row y run the rounds of pool y and
// never look at another row.  A round of one pool is a chain of L2 round trips (count exchange, store -> poll) with
// little work in between; two co-resident CTAs per SM working on different pools fill each other's waits.
struct LlMultiParams {
  LlParams pool[LL_MAX_POOLS];
};

// ---- named barriers of the persistent kernel: LL_BAR_W among the worker warps only, LL_BAR_SCAN workers -> exchange
// warp (bar.arrive / bar.sync: the counts are scanned), LL_BAR_HAND exchange warp <-> workers (the handoff, and the
// start and the end of the kernel).  The second half of a two-pool CTA uses the same three ids + LL_BAR_HALF.
constexpr int LL_BAR_W = 1, LL_BAR_SCAN = 2, LL_BAR_HAND = 3, LL_BAR_HALF = 3;
__device__ __forceinline__ void ll_arrive(int id, int threads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
__device__ __forceinline__ void ll_wait(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
__device__ __forceinline__ bool ll_bar_or(int id, int threads, bool pred) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "bar.red.or.pred q, %2, %3, p;\n\t"
      "selp.u32 %0, 1, 0, q;\n\t}"
      : "=r"(r)
      : "r"(static_cast<uint32_t>(pred)), "r"(id), "r"(threads)
      : "memory");
  return r != 0;
}
__device__ __forceinline__ void ld_fat2(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
// (no "memory" clobber: the compiler may move the shared-memory loads that feed later stores across this one)
__device__ __forceinline__ void st_fat2(unsigned long long* p, unsigned long long a, unsigned long long b) {
  asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b));
}

// ---- plain arena <-> fat arena (one thread per node; not performance critical: the whole pool, once per hand-over).
// Byte for byte for every node tsb_nq_pool_push admits (depth <= N, board[0..N) < N, bytes past N zero), which
// are the only nodes a pool holds.

// a node's word of the earlier 64-byte format, from its board by the reference predicate, row by row:
//   bits  0..19  ld: values attacked on the node's next row along the rising diagonals  {board[i] + (depth - i)}
//   bits 20..39  rd: ... along the falling diagonals                                     {board[i] - (depth - i)}
//   bits 40..59  the node's child mask: slot k set <=> k >= depth and board[k] is not attacked (evaluate_gpu's
//                label for slot k, nqueens_gpu_chpl.chpl:97-123)
//   bit  60      leaf (depth == N)
__device__ __forceinline__ unsigned long long nq_aux_pack(uint32_t ld, uint32_t rd, uint32_t cm, bool leaf) {
  return static_cast<unsigned long long>(ld) | static_cast<unsigned long long>(rd) << 20 |
         static_cast<unsigned long long>(cm) << 40 | static_cast<unsigned long long>(leaf ? 1u : 0u) << 60;
}
template <int N>
__device__ __forceinline__ unsigned long long nq_aux_of_node(const uint8_t* node) {
  const int d = node[0];
  uint32_t ld = 0, rd = 0;
  for (int i = 0; i < d && i < N; i++) {
    const int b = node[1 + i], s = d - i;
    if (b + s < N) ld |= 1u << (b + s);
    if (b - s >= 0) rd |= 1u << (b - s);
  }
  const uint32_t U = ld | rd;
  uint32_t cm = 0;
  for (int k = d; k < N; k++)
    if (!((U >> (node[1 + k] & 31)) & 1u)) cm |= 1u << k;
  return nq_aux_pack(ld, rd, cm, d == N);
}
// (tag 0: the nodes are the trusted layer of the next launch)
template <int N>
__global__ void nq_fat_import_kernel(const uint8_t* __restrict__ arena, FatNode* __restrict__ fat, long long size) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= size) return;
  const uint8_t* node = arena + p * NQ_REC;
  uint32_t d[LL_WORDS] = {0, 0, 0, 0};
  for (int i = 0; i < NQ_REC - 1; i++) d[ll_fw(i)] |= static_cast<uint32_t>(node[1 + i]) << ll_fs(i);
  ll_set_depth(d, node[0]);
  const unsigned long long aux = nq_aux_of_node<N>(node);
  d[3] |= (static_cast<uint32_t>(aux >> 40) & 0xFFFFFu) << LL_CM_SHIFT | ((aux >> 60) & 1u ? LL_LEAF : 0u);
  unsigned long long w[LL_WORDS];
  ll_piece(d[0], d[1], static_cast<uint32_t>(aux) & 0xFFFFFu, 0u, w[0], w[1]);
  ll_piece(d[2], d[3], static_cast<uint32_t>(aux >> 20) & 0xFFFFFu, 0u, w[2], w[3]);
  for (int i = 0; i < LL_WORDS; i += 2) st_fat2(&fat[p].w[i], w[i], w[i + 1]);
}
// the same for 25-byte records: board[18..23] in data32[3], no child mask or leaf flag, the diagonal masks N <= 24
// bits each.  (A kernel of its own: as a template over the record width the 21-byte kernel's SASS would not stay the
// same.)
template <int N>
__global__ void nq_fat_import_wide_kernel(const uint8_t* __restrict__ arena, FatNode* __restrict__ fat, long long size) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= size) return;
  const uint8_t* node = arena + p * NQ_REC24;
  uint32_t d[LL_WORDS] = {0, 0, 0, 0};
  for (int i = 0; i < NQ_REC24 - 1; i++) d[ll_fw(i)] |= static_cast<uint32_t>(node[1 + i]) << ll_fs(i);
  ll_set_depth(d, node[0]);
  const int depth = node[0];
  uint32_t ld = 0, rd = 0;
  for (int i = 0; i < depth && i < N; i++) {
    const int b = node[1 + i], s = depth - i;
    if (b + s < N) ld |= 1u << (b + s);
    if (b - s >= 0) rd |= 1u << (b - s);
  }
  unsigned long long w[LL_WORDS];
  ll_piece(d[0], d[1], ld, 0u, w[0], w[1]);
  ll_piece(d[2], d[3], rd, 0u, w[2], w[3]);
  for (int i = 0; i < LL_WORDS; i += 2) st_fat2(&fat[p].w[i], w[i], w[i + 1]);
}
// the clear: tag 0 on the `words` first words of the arena, data kept
__global__ void nq_fat_clear_tags_kernel(FatNode* __restrict__ fat, long long words) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < words) {
    unsigned long long* w = &fat[0].w[0] + i;
    *w &= 0x0000FFFFFFFFFFFFull;
  }
}
// fat nodes -> R-byte records (nq_fat_export_kernel, nq_fat_export_wide_kernel)
template <int R>
__device__ __forceinline__ void nq_fat_export_body(const FatNode* __restrict__ fat, uint8_t* __restrict__ arena, long long size) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= size) return;
  uint8_t* node = arena + p * R;
  uint32_t d[LL_WORDS];
  for (int i = 0; i < LL_WORDS; i++) d[i] = static_cast<uint32_t>(fat[p].w[i]);
  node[0] = static_cast<uint8_t>(ll_depth(d[0], d[1], d[2]));
  for (int i = 0; i < R - 1; i++) node[1 + i] = static_cast<uint8_t>(d[ll_fw(i)] >> ll_fs(i) & 31u);
}
__global__ void nq_fat_export_kernel(const FatNode* __restrict__ fat, uint8_t* __restrict__ arena, long long size) {
  nq_fat_export_body<NQ_REC>(fat, arena, size);
}
__global__ void nq_fat_export_wide_kernel(const FatNode* __restrict__ fat, uint8_t* __restrict__ arena, long long size) {
  nq_fat_export_body<NQ_REC24>(fat, arena, size);
}

// The exchange warp's count gather: 2G slots {epoch << 32 | leaves << 20 | children}, lane l holds the slot pairs
// 2l + 64u.  Its first LL_GB pairs are loaded back to back, so a sweep over up to 64 LL_GB slots (2G on GPUs of up to
// 160 SMs) is ONE L2 round trip.  (A loop that summed each pair before it loaded the next one issued them one after
// the other: two or three dependent round trips per sweep at 2G = 132, all of the last sweep exposed in the round.)
// Further pairs (more than 160 CTAs per pool) are loaded one by one.
constexpr int LL_GB = 5;
__device__ __forceinline__ void ll_load_pair(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
static_assert(64 * LL_GB <= 2 * LL_MAX_SMS, "a lane's first LL_GB pairs lie inside LlSync::slot");
__device__ __forceinline__ bool ll_pair_carries(int n, int i, unsigned epoch, unsigned long long a, unsigned long long b) {
  return static_cast<unsigned>(a >> 32) == epoch && (i + 1 >= n || static_cast<unsigned>(b >> 32) == epoch);
}
// Which of the lane's first 2 LL_GB slots (bit 2u + e: slot 2 lane + 64u + e) exist and lie before k0 / k1.  They are
// the same in every round, so a sweep and the sums test bits instead of comparing slot numbers.
struct LlLaneSlots {
  unsigned in, lt0, lt1;
};
__device__ __forceinline__ LlLaneSlots ll_lane_slots(int n, int k0, int k1) {
  const int c0 = 2 * (threadIdx.x & 31);
  LlLaneSlots m = {0u, 0u, 0u};
#pragma unroll
  for (int j = 0; j < 2 * LL_GB; j++) {
    const int i = c0 + 64 * (j >> 1) + (j & 1);
    m.in |= (i < n ? 1u : 0u) << j;
    m.lt0 |= (i < k0 ? 1u : 0u) << j;
    m.lt1 |= (i < k1 ? 1u : 0u) << j;
  }
  // (opaque to the compiler: the masks stay in three registers instead of being recomputed from the compares in
  // every round's sums)
  asm volatile("" : "+r"(m.in), "+r"(m.lt0), "+r"(m.lt1));
  return m;
}
// Sweeps until all n slots carry `epoch`; the lane's first LL_GB pairs of the sweep that saw every slot stay in v0 /
// v1.  A sweep only tests the epochs: the sums run once, after it (warp_sum_slots2).  `in_flight()` runs once, while
// the first sweep's loads are on their way.  false = abort.  (Group u is skipped by the whole warp when 64u >= n; in
// a group that is loaded, a lane past n loads a slot inside the array and ignores it.)
template <class F>
__device__ __forceinline__ bool warp_gather_slots2(const unsigned long long* slot, int n, unsigned epoch,
                                                   unsigned* abort_flag, const LlLaneSlots& ls,
                                                   unsigned long long (&v0)[LL_GB], unsigned long long (&v1)[LL_GB],
                                                   F&& in_flight) {
  const int c0 = 2 * (threadIdx.x & 31);
  const auto load = [&]() {
#pragma unroll
    for (int u = 0; u < LL_GB; u++)
      if (64 * u < n) ll_load_pair(slot + c0 + 64 * u, v0[u], v1[u]);
  };
  SpinGuard guard;
  load();
  in_flight();
  for (;;) {
    bool ok = true;
#pragma unroll
    for (int u = 0; u < LL_GB; u++)
      if (64 * u < n)
        ok &= (static_cast<unsigned>(v0[u] >> 32) == epoch || !(ls.in >> (2 * u) & 1u)) &&
              (static_cast<unsigned>(v1[u] >> 32) == epoch || !(ls.in >> (2 * u + 1) & 1u));
    for (int i = c0 + 64 * LL_GB; i < n; i += 64) {
      unsigned long long a, b;
      ll_load_pair(slot + i, a, b);
      ok &= ll_pair_carries(n, i, epoch, a, b);
    }
    if (__all_sync(0xFFFFFFFFu, ok)) return true;
    if (__any_sync(0xFFFFFFFFu, guard.expired(abort_flag))) return false;
    load();
  }
}
// The gathered children over all slots and over the slots before k0 / k1 (in every lane: at most 2G x 18 432, 32
// bits), and this lane's share of the leaves
__device__ __forceinline__ void warp_sum_slots2(const unsigned long long* slot, const unsigned long long (&v0)[LL_GB],
                                                const unsigned long long (&v1)[LL_GB], int n, int k0, int k1,
                                                const LlLaneSlots& ls, unsigned& all, unsigned& before0,
                                                unsigned& before1, unsigned& leaves) {
  const int c0 = 2 * (threadIdx.x & 31);
  all = before0 = before1 = leaves = 0;
  const auto add = [&](unsigned x, bool in, bool lt0, bool lt1) {
    x = in ? x : 0u;
    const unsigned y = x & 0xFFFFFu;
    all += y;
    leaves += x >> 20;
    before0 += lt0 ? y : 0u;
    before1 += lt1 ? y : 0u;
  };
#pragma unroll
  for (int u = 0; u < LL_GB; u++)
    if (64 * u < n) {
      add(static_cast<unsigned>(v0[u]), ls.in >> (2 * u) & 1u, ls.lt0 >> (2 * u) & 1u, ls.lt1 >> (2 * u) & 1u);
      add(static_cast<unsigned>(v1[u]), ls.in >> (2 * u + 1) & 1u, ls.lt0 >> (2 * u + 1) & 1u, ls.lt1 >> (2 * u + 1) & 1u);
    }
  // (further pairs are loaded again: they still hold this round's values, because another CTA writes this parity's
  // slots again two rounds on, after it has seen this CTA's slots of the next round)
  for (int i = c0 + 64 * LL_GB; i < n; i += 64) {
    unsigned long long a, b;
    ll_load_pair(slot + i, a, b);
    add(static_cast<unsigned>(a), true, i < k0, i < k1);
    add(static_cast<unsigned>(b), i + 1 < n, i + 1 < k0, i + 1 < k1);
  }
  // (three independent warp reductions, redux.sync)
  all = __reduce_add_sync(0xFFFFFFFFu, all);
  before0 = __reduce_add_sync(0xFFFFFFFFu, before0);
  before1 = __reduce_add_sync(0xFFFFFFFFu, before1);
}

// what the exchange warp hands the workers at the end of a round's gather (one record: the workers copy the offsets
// right after the handoff and the geometry before their next poll; the exchange warp writes the next record only
// after the next scan, i.e. after both)
struct LlPlan {
  long long s0;             // next round: position of the chunk's first parent (= of the round's first child)
  int a0, len0, a1, len1;   // next round: this CTA's two sub-slices of the chunk (first parent, parents)
  unsigned tag;             // next round's tag (ll_tag of its epoch)
  int top;                  // next round: top layer of the layer stack
  int exit;                 // -1: run the next round; else the RND_EXIT_* code all threads leave with
  int off0, off1;           // this round: first child of each of this CTA's sub-slices among the round's children
};
// TSB200_ROUNDS_PROF phases (CTA 0 cycles; workers: thread 0, exchange warp: its lane 0)
enum {
  LL_PROF_SETUP = 0, LL_PROF_POLL, LL_PROF_SCAN, LL_PROF_BUILD, LL_PROF_HAND, LL_PROF_STORE,  // workers
  LL_PROF_X_SCAN, LL_PROF_X_AHEAD, LL_PROF_X_GATHER, LL_PROF_X_TAIL, LL_PROF_X_HAND,        // exchange warp
  LL_PROF_N
};
static_assert(LL_PROF_N <= 12, "RoundsState::prof");
// (R: the pool's record width; a parent has at most R - 1 children)
template <int T, int PPT, int R = NQ_REC>
struct LlSmem {
  alignas(16) uint4 parent[T * PPT];   // the slice: data32[0..3] of every parent
  alignas(8) uint2 diag[T * PPT];      // ... and its {ld, rd}
  alignas(16) uint4 stage[LL_CAP];     // the window's children: data32[0..3]
  alignas(8) uint2 stage_diag[LL_CAP]; // ... and their {ld, rd}
  alignas(16) uint16_t item[T * PPT * (R - 1)];  // (record << 5) | slot, in child order
  unsigned long long warp_tot64[T / 32];
  LlPlan plan;
  int poll_abort;                  // a worker's poll gave up: the exchange warp leaves after the scan barrier
  long long prof[LL_PROF_N], prof_t[2];  // (prm.prof, CTA 0) cycles per phase; clock at the end of the last one
                                         // (workers, exchange warp)
  unsigned prof_fertile, prof_wide;  // (prm.prof, every CTA) parents with children; rounds of more than one window
  long long lay_start[LL_LAYERS];  // the pool's layers, bottom to top: first position ...
  unsigned lay_tag[LL_LAYERS];     // ... and the tag its nodes were stored with (LL_TRUSTED: before the launch)
};

// The child mask of a node with data words P at `depth` whose row `depth` has the safe values S = ~(ld | rd): slot i
// set <=> i >= depth and bit board[i] of S is set (evaluate_gpu's label for slot i).  Only the data words that hold a
// slot >= depth are read (word 0 is skipped from depth 6 on, word 1 from depth 12, word 2 from depth 18); the slots of
// the words that are read are masked at the end (none for a leaf).  Bits of P above the board are ignored.
template <int N>
__device__ __forceinline__ uint32_t ll_child_mask(const uint32_t (&P)[4], uint32_t depth, uint32_t S) {
  uint32_t cm = 0;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    if (6 * j >= N) break;
    if (6 * j + 6 < N && depth >= static_cast<uint32_t>(6 * j + 6)) continue;
#pragma unroll
    for (int i = 6 * j; i < 6 * j + 6 && i < N; i++) {
      const uint32_t x = shf_r_wrap(S, 0u, P[j] >> ll_fs(i)) & 1u;  // bit board[i] of S (the shift wraps mod 32)
      asm("mad.lo.u32 %0, %1, %2, %0;" : "+r"(cm) : "r"(x), "r"(1u << i));  // cm |= x << i on the FMA pipe
    }
  }
  return cm & shl_clamp(0xFFFFFFFFu, depth);
}

// child `item` of the slice -> its four data words (board[depth] and board[k] swapped, depth + 1; 21-byte records: its
// child mask evaluated here, ll_child_mask) and *cdiag its diagonal masks, from its parent's
template <int N, int R>
__device__ __forceinline__ uint4 ll_build_child(const uint4* parent, const uint2* diag, int item, uint2* cdiag) {
  const int r = item >> 5;
  const uint32_t k = static_cast<uint32_t>(item & 31);
  const uint4 p = parent[r];
  uint32_t P[4] = {p.x, p.y, p.z, p.w};
  const uint32_t depth = ll_depth(p.x, p.y, p.z);
  // first bit of board[i] in the four data words read as one 128-bit value: 32 (i / 6) + 5 (i % 6) = 5 i + 2 (i / 6),
  // with i / 6 = (43 i) >> 8 for every i < 24 (no division; it holds up to i = 127)
  const uint32_t bd = 5u * depth + 2u * (depth * 43u >> 8), bk = 5u * k + 2u * (k * 43u >> 8);
  // (a clamped right shift by b - 32 j is the field at bit b in word j and 0 in every other word)
  const auto field = [&](uint32_t b) {
    return (shr_clamp(P[0], b) | shr_clamp(P[1], b - 32u) | shr_clamp(P[2], b - 64u) | shr_clamp(P[3], b - 96u)) & 31u;
  };
  const uint32_t v = field(bk);  // the queen placed on row `depth`
  const uint32_t D = field(bd) ^ v;
  // (a clamped shift by bd - 32 j is D << sd in word wd and 0 in every other word: no field straddles two words)
#pragma unroll
  for (uint32_t j = 0; j < 4; j++) P[j] ^= shl_clamp(D, bd - 32u * j) ^ shl_clamp(D, bk - 32u * j);
  const uint32_t cd = depth + 1u;
  ll_set_depth(P, cd);
  const uint2 pd = diag[r];
  const uint32_t bit = 1u << v;
  const uint32_t cld = ((pd.x | bit) << 1) & ((1u << N) - 1u), crd = (pd.y | bit) >> 1;
  *cdiag = make_uint2(cld, crd);
  if constexpr (R == NQ_REC) {
    const uint32_t cm = ll_child_mask<N>(P, cd, ~(cld | crd));  // (the safe values of row cd)
    P[3] = (P[3] & 0x3FFu) | cm << LL_CM_SHIFT | (cd == static_cast<uint32_t>(N) ? LL_LEAF : 0u);
  }
  // (25-byte records: data32[3] is board[18..23], bits 30..31 stay 0)
  return make_uint4(P[0], P[1], P[2], P[3]);
}

// One CTA = LL_T worker threads (warps 0-7) + one EXCHANGE warp (warp 8).  A round:
//   workers:   poll the slice -> child masks, block scan -> (LL_BAR_SCAN arrive) -> items -> build the first window
//              -> HANDOFF -> store the windows -> the next round's poll
//   exchange:  (LL_BAR_SCAN wait) -> publish the CTA's two count slots -> issue the first sweep over all 2G slots ->
//              while it is in flight: layer-stack pop and new top entry, next tag and top layer, the interval of the
//              round's total R for which the next round is plan()'s common case -> sweeps that only test epochs ->
//              sums of the last sweep (offsets, R) -> common case: next chunk start; else plan() -> HANDOFF ->
//              counters
// so the gather runs while the workers build, and the bookkeeping of a round and the set-up of the next are off the
// workers' chain: after their stores they go straight into the next poll.  Between the last slot's arrival and the
// handoff only the sums, a range test and a few shared-memory stores remain.  The pool state (size, epoch, layers,
// counters) is the exchange warp's alone; the workers get what they need through sm.plan.
//
// HALVES = 2 (four pools per launch): a CTA of 2 (T + 32) threads runs two pools, one per HALF, so no pool is the
// second CTA on its SMs.  Half h is threads [h TX, (h + 1) TX) = warps 9h .. 9h + 8 and runs pool blockIdx.y + 2h
// exactly as a CTA of HALVES = 1 would: its own LlSmem (the second right after the first), its own barrier ids
// (+ LL_BAR_HALF), no barrier over the whole CTA; a half whose pool has left has exited.  Pools 0 + 2 and 1 + 3 share
// a CTA: in the steps where pools run dry (the host's steals), 0 and 1 or 2 and 3 leave early together, and the two
// that run on then hold one SM each, where pairs 0 + 1 / 2 + 3 would leave them sharing half the SMs while the other
// half idles (DESIGN §5).  The warps of an SM's
// sub-partition are those of equal warp id mod 4: nine warps per half put both halves' warps on every sub-partition,
// two workers of each half on each, the exchange warps (8 and 17) on sub-partitions 0 and 1.  With two CTAs per SM the
// CTA that became resident second ran the slower pool (DESIGN §5).
//
// REC: the record width of the pool's plain arena, which decides the fat node's data32[3] (see the top of this file):
// NQ_REC (nq_rounds_ll_kernel, every variant) or NQ_REC24 (nq_rounds_ll_wide_kernel: one pool per launch).
template <int N, int T, int PPT, int HALVES, int REC>
__device__ __forceinline__ void nq_rounds_ll_body(const LlMultiParams& mprm) {
  constexpr int LL_PPT = PPT;
  constexpr int TX = T + 32;  // the whole CTA (HALVES = 1) or half: workers + exchange warp
  const int half = HALVES == 2 && threadIdx.x >= TX ? 1 : 0;
  const LlParams& prm = mprm.pool[blockIdx.y + gridDim.y * half];
  extern __shared__ __align__(128) uint8_t smem_raw[];
  LlSmem<T, PPT, REC>& sm = reinterpret_cast<LlSmem<T, PPT, REC>*>(smem_raw)[half];
  const int bar_w = LL_BAR_W + LL_BAR_HALF * half, bar_scan = LL_BAR_SCAN + LL_BAR_HALF * half,
            bar_hand = LL_BAR_HAND + LL_BAR_HALF * half;
  const int t = threadIdx.x - TX * half, lane = t & 31, wid = t >> 5;
  const int k = blockIdx.x, G = gridDim.x, G2 = 2 * G;
  LlSync* const sy = prm.sync;
  FatNode* const fat = prm.fat;
  // the profile lives in shared memory, touched by CTA 0's thread 0 (workers) and thread T (exchange warp) only: no
  // per-thread state, nothing when it is off
  const bool prof_w = prm.prof != 0 && k == 0 && t == 0;
  const bool prof_x = prm.prof != 0 && k == 0 && t == T;
#define TSB_PROF(on, who, i)          \
  if (on) {                           \
    const long long now = clock64();  \
    sm.prof[i] += now - sm.prof_t[who]; \
    sm.prof_t[who] = now;             \
  }

  // ---- the exchange warp's pool state (every lane holds the same values; lane 0 writes shared memory)
  long long size = prm.size0, chunk_s0 = 0, chunk_n = 0;  // (the chunk of the current round)
  long long size_hi = prm.size0;
  unsigned epoch = prm.epoch0;
  int n_lay = prm.size0 > 0 ? 1 : 0;
  long long lay_top = 0;  // lay_start[n_lay - 1] (n_lay > 0)
  unsigned long long rounds = 0, tot_parents = 0, tot_children = 0, tot_solutions = 0;
  int exit_code = RND_EXIT_PAUSE;
  // this CTA's sub-slices of a chunk of geo_n parents (relative to the chunk's start: they depend on n alone, and
  // n == M in almost every round, so the four divisions run only when n changes)
  long long geo_n = -1;
  int geo_a0 = 0, geo_len0 = 0, geo_a1 = 0, geo_len1 = 0;
  // (0) the next round's chunk: popBackBulk(m, M) -> sm.plan; -1 or the exit code (uniform decisions: every CTA
  // holds the same state)
  const auto plan = [&]() {
    int ex = -1;
    if (size < prm.m)
      ex = RND_EXIT_DONE;
    else if (static_cast<long long>(rounds) >= prm.max_rounds)
      ex = RND_EXIT_PAUSE;
    else {
      chunk_n = size < prm.M ? size : prm.M;
      chunk_s0 = size - chunk_n;
      if (chunk_s0 + chunk_n * N > prm.cap)  // worst case: every slot of every parent survives
        ex = RND_EXIT_SPACE;
      // (no room to record this round's children, or no epoch left whose tag cannot alias: start over with one
      // trusted layer)
      else if (n_lay >= LL_LAYERS || epoch == prm.epoch_last)
        ex = RND_EXIT_RELAUNCH;
    }
    if (ex < 0) {
      ++epoch;
      // this CTA's share of the chunk: TWO sub-slices of n / 2G parents — number k from the bottom and number k from
      // the top.  The bottom of a chunk holds the shallow nodes (many children), the top the deep ones (few): a
      // single slice per CTA left the bottom CTA with 3x the average children, and its build + node stores were the
      // round's critical path; pairing k with 2G-1-k evens the load without knowing it in advance.
      // (n <= 768 G and k < G <= 256: the products fit 32 bits — 64-bit divisions are slow emulated sequences)
      if (chunk_n != geo_n) {
        geo_n = chunk_n;
        const unsigned n32 = static_cast<unsigned>(chunk_n), uG2 = static_cast<unsigned>(G2), uk = static_cast<unsigned>(k);
        geo_a0 = static_cast<int>(n32 * uk / uG2);
        geo_len0 = static_cast<int>(n32 * (uk + 1u) / uG2) - geo_a0;
        geo_a1 = static_cast<int>(n32 * (uG2 - 1u - uk) / uG2);
        geo_len1 = static_cast<int>(n32 * (uG2 - uk) / uG2) - geo_a1;
      }
      if (lane == 0) {
        sm.plan.s0 = chunk_s0;
        sm.plan.a0 = geo_a0;
        sm.plan.len0 = geo_len0;
        sm.plan.a1 = geo_a1;
        sm.plan.len1 = geo_len1;
        sm.plan.tag = ll_tag(epoch);
        sm.plan.top = n_lay - 1;
      }
    }
    if (lane == 0) sm.plan.exit = ex;
    return ex;
  };

  if (wid == T / 32) {
    if (lane == 0) {
      sm.lay_start[0] = 0;
      sm.lay_tag[0] = LL_TRUSTED;
      sm.poll_abort = 0;
      sm.prof_fertile = sm.prof_wide = 0;
      if (prm.prof != 0) {
        const unsigned long long now = ll_globaltimer();
        prm.state->cta_sm[k] = ll_smid();
        prm.state->cta_t0[k] = static_cast<unsigned>(now);
        if (k == 0) prm.state->t_start = now;
      }
      if (prof_x)
        for (int i = 0; i < LL_PROF_N; i++) sm.prof[i] = 0;
    }
    exit_code = plan();
  }
  ll_bar_or(bar_hand, TX, false);  // (sm.plan of the first round)
  if (prm.prof != 0 && k == 0 && (t == 0 || t == T)) sm.prof_t[t == T] = clock64();

  if (wid == T / 32) {
    // ------------------------------------------------------------------------------------------ the exchange warp
    const LlLaneSlots lane_slots = ll_lane_slots(G2, k, G2 - 1 - k);
    while (exit_code < 0) {
      ll_wait(bar_scan, TX);  // the workers' warp totals are in sm.warp_tot64 (they have read their slices)
      TSB_PROF(prof_x, 1, LL_PROF_X_SCAN)
      if (sm.poll_abort) {
        exit_code = RND_EXIT_ABORT;
        break;
      }
      // ---- (4) publish {epoch, leaves, children} of my two sub-slices (slot s = sub-slice s, bottom to top)
      unsigned long long tot = 0;
#pragma unroll
      for (int i = 0; i < T / 32; i++) tot += sm.warp_tot64[i];
      const unsigned my_children = static_cast<unsigned>(tot & 0xFFFFF), my_leaves = static_cast<unsigned>(tot >> 20) & 0xFFFu;
      const unsigned cnt0 = static_cast<unsigned>(tot >> 32) & 0xFFFFFu;
      unsigned long long* const slots = sy->slot[epoch & 1u];
      const unsigned long long e = static_cast<unsigned long long>(epoch) << 32;
      if (lane < 2)
        st_relaxed_u64(&slots[lane == 0 ? k : G2 - 1 - k],
                       lane == 0 ? e | static_cast<unsigned long long>(my_leaves) << 20 | cnt0 : e | (my_children - cnt0));
      // ---- (6) all-to-all: everybody's {leaves, children} (the workers build their first window meanwhile).
      // While the first sweep's loads are on their way, everything of the round's bookkeeping that does not depend
      // on its total R of children:
      // (8) the pool's layers after the round: every layer that starts inside the chunk is consumed, the round's
      // children form the new top layer (same computation in every CTA).  The workers read the stack only in their
      // poll, and all of them have finished this round's poll (they arrived at LL_BAR_SCAN) and start the next one
      // after the handoff: nobody reads an entry while it changes.  So the new top entry is written now; if R == 0 it
      // lies above the top the stack keeps (nl entries) and is never read.  (lay_top = lay_start[n_lay - 1]: the loop
      // ends at the top layer in most rounds, without waiting for a shared-memory load.)
      // (9) the next round's tag and top layer for the common case, straight into sm.plan: the workers read them
      // before their poll, i.e. before LL_BAR_SCAN this round and after the handoff next round; if plan() runs
      // instead it writes them again.  And the interval of R for which plan() would take the common case: the pool
      // keeps at least max(M, m) nodes, so the next chunk is M == geo_n parents and its geometry stands, and no exit
      // applies (arena room for the next chunk's children, round budget, layer table, epoch window).
      const long long n_prev = chunk_n;
      int nl = n_lay;
      long long below = lay_top, r_lo = 1, r_hi = 0;
      const auto plan_ahead = [&]() {
        while (nl > 0 && below >= chunk_s0) {
          --nl;
          below = nl > 0 ? sm.lay_start[nl - 1] : -1;
        }
        __syncwarp();  // (every lane has read the entry lane 0 may overwrite)
        if (lane == 0) {
          sm.lay_start[nl] = chunk_s0;
          sm.lay_tag[nl] = ll_tag(epoch);
          sm.plan.tag = ll_tag(epoch + 1u);
          sm.plan.top = nl;
        }
        const long long Mx = prm.M > prm.m ? prm.M : prm.m;
        r_lo = Mx - chunk_s0 > 1 ? Mx - chunk_s0 : 1;  // (R > 0: the new top layer exists)
        if (geo_n == prm.M && static_cast<long long>(rounds) + 1 < prm.max_rounds && nl + 1 < LL_LAYERS &&
            epoch != prm.epoch_last)
          r_hi = prm.cap - static_cast<long long>(prm.M) * N + prm.M - chunk_s0;  // (chunk_s0 + R - M) + M N <= cap
        TSB_PROF(prof_x, 1, LL_PROF_X_AHEAD)
      };
      unsigned long long v0[LL_GB], v1[LL_GB];
      const bool ok = warp_gather_slots2(slots, G2, epoch, &sy->abort, lane_slots, v0, v1, plan_ahead);
      TSB_PROF(prof_x, 1, LL_PROF_X_GATHER)
      unsigned R = 0, leaves = 0;
      if (ok) {
        // my child offsets and the round's total; then the rest of (8) and (9)
        unsigned before0, before1;
        warp_sum_slots2(slots, v0, v1, G2, k, G2 - 1 - k, lane_slots, R, before0, before1, leaves);
        if (lane == 0) {
          sm.plan.off0 = static_cast<int>(before0);
          sm.plan.off1 = static_cast<int>(before1);
        }
        ++rounds;
        size = chunk_s0 + R;
        n_lay = R > 0 ? nl + 1 : nl;
        lay_top = R > 0 ? chunk_s0 : below;
        if (R >= r_lo && R <= r_hi) {  // plan()'s common case: chunk_n, the geometry, tag, top and exit stand
          ++epoch;
          chunk_s0 = size - chunk_n;
          if (lane == 0) sm.plan.s0 = chunk_s0;
        } else {
          exit_code = plan();
        }
      }
      TSB_PROF(prof_x, 1, LL_PROF_X_TAIL)
      if (ll_bar_or(bar_hand, TX, !ok)) {  // the handoff (an abort reaches the workers here)
        exit_code = RND_EXIT_ABORT;
        break;
      }
      TSB_PROF(prof_x, 1, LL_PROF_X_HAND)
      // the round's counters, after the handoff
      size_hi = size > size_hi ? size : size_hi;
      tot_parents += static_cast<unsigned long long>(n_prev);
      tot_children += R;
      tot_solutions += __reduce_add_sync(0xFFFFFFFFu, leaves);
    }
    if (prof_x) prm.state->t_exit = ll_globaltimer();
  } else {
    // ------------------------------------------------------------------------------------------ the workers
    unsigned prof_fertile = 0;  // (prm.prof) parents of this thread's records that had children
    for (;;) {
      if (sm.plan.exit >= 0) break;
      const long long s0 = sm.plan.s0;
      const int a0 = sm.plan.a0, len0 = sm.plan.len0, a1 = sm.plan.a1, len1 = sm.plan.len1;
      const unsigned round_tag = sm.plan.tag;
      const int top = sm.plan.top;
      const int len = len0 + len1;
      bool ok = true;
      TSB_PROF(prof_w, 0, LL_PROF_SETUP)

      // ---- (2) my slice -> shared memory, 16-byte piece by piece (2 pieces per node, consecutive lanes on
      // consecutive pieces: every warp load is 512 contiguous bytes); a piece is polled until both of its words
      // carry the tag of the layer its node lies in
      {
        SpinGuard guard;
        const unsigned long long* src0 = fat[s0 + a0].w;
        const unsigned long long* src1 = fat[s0 + a1].w - LL_WORDS * len0;  // (indexed by the concatenated piece number)
        constexpr int PCS = 2 * LL_PPT;  // pieces per thread
        unsigned long long w0[PCS], w1[PCS];
        unsigned pending = 0;
#pragma unroll
        for (int j = 0; j < PCS; j++)
          if (t + j * T < 2 * len) pending |= 1u << j;
        // the tag node i of my slice was stored with: that of the layer its position lies in (mostly the top one)
        // (in almost every round both sub-slices lie in the top layer: then every piece is checked against one tag in a
        // register, and the sweeps make no shared-memory loads of the stack)
        const long long top_start = sm.lay_start[top];
        const unsigned top_tag = sm.lay_tag[top];
        const bool in_top = s0 + min(a0, a1) >= top_start;
        const auto want_of = [&](int i) {
          if (in_top) return top_tag;
          const long long pos = s0 + (i < len0 ? a0 + i : a1 + (i - len0));
          int L = top;
          while (L > 0 && sm.lay_start[L] > pos) --L;
          return sm.lay_tag[L];
        };
        while (pending) {
          // all loads of a sweep are issued back to back (a dependent re-poll per piece would serialise 8 L2 round
          // trips)
#pragma unroll
          for (int j = 0; j < PCS; j++)
            if (pending & (1u << j)) {
              const int pc = t + j * T;
              ld_fat2((pc < 2 * len0 ? src0 : src1) + 2 * pc, w0[j], w1[j]);
            }
#pragma unroll
          for (int j = 0; j < PCS; j++)
            if (pending & (1u << j)) {
              const int pc = t + j * T, i = pc >> 1;
              const unsigned want = want_of(i);
              const uint32_t h0 = static_cast<uint32_t>(w0[j] >> 32), h1 = static_cast<uint32_t>(w1[j] >> 32);
              if (want == LL_TRUSTED || __byte_perm(h0, h1, 0x7632) == want * 0x10001u) {  // (both tags)
                reinterpret_cast<uint2*>(sm.parent)[pc] = make_uint2(static_cast<uint32_t>(w0[j]), static_cast<uint32_t>(w1[j]));
                reinterpret_cast<uint32_t*>(sm.diag)[pc] = __byte_perm(h0, h1, 0x5410);  // ld or rd
                pending &= ~(1u << j);
              }
            }
          if (pending && guard.expired(&sy->abort)) {
            ok = false;
            break;
          }
        }
      }
      if (ll_bar_or(bar_w, T, !ok)) {  // the slice is in shared memory
        if (t == 0) sm.poll_abort = 1;
        ll_arrive(bar_scan, TX);  // (the exchange warp waits there, sees the flag and leaves too)
        break;
      }
      uint32_t cm[LL_PPT];
      int leaves = 0, mine = 0, mine0 = 0;
#pragma unroll
      for (int q = 0; q < LL_PPT; q++) {
        const int i = LL_PPT * t + q;
        cm[q] = 0;
        if (i < len) {
          if constexpr (REC == NQ_REC) {
            const uint32_t w3 = sm.parent[i].w;
            cm[q] = w3 >> LL_CM_SHIFT & 0xFFFFFu;
            leaves += (w3 & LL_LEAF) ? 1 : 0;
          } else {  // (no stored mask or leaf flag: evaluated from the board, the depth and the diagonal masks)
            const uint4 p = sm.parent[i];
            const uint2 dg = sm.diag[i];
            const uint32_t P[4] = {p.x, p.y, p.z, p.w}, depth = ll_depth(p.x, p.y, p.z);
            cm[q] = ll_child_mask<N>(P, depth, ~(dg.x | dg.y));
            leaves += depth == static_cast<uint32_t>(N) ? 1 : 0;
          }
          mine += __popc(cm[q]);
          if (i < len0) mine0 += __popc(cm[q]);
        }
      }
      TSB_PROF(prof_w, 0, LL_PROF_POLL)
      if (prm.prof != 0)
#pragma unroll
        for (int q = 0; q < LL_PPT; q++) prof_fertile += cm[q] != 0u ? 1u : 0u;
      // ---- (3) block scan: children | leaves << 20 | children of the bottom sub-slice << 32 (at most 768 x 24 =
      // 18 432, 768 and 18 432 per CTA: no field overflows into the next)
      unsigned long long incl = static_cast<unsigned long long>(mine) | static_cast<unsigned long long>(leaves) << 20 |
                                static_cast<unsigned long long>(mine0) << 32;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= o) incl += y;
      }
      if (lane == 31) sm.warp_tot64[wid] = incl;
      ll_arrive(bar_scan, TX);  // the exchange warp publishes the totals and gathers everybody's
      ll_wait(bar_w, T);
      unsigned long long woff = 0, tot = 0;
#pragma unroll
      for (int i = 0; i < T / 32; i++) {
        if (i < wid) woff += sm.warp_tot64[i];
        tot += sm.warp_tot64[i];
      }
      const int my_children = static_cast<int>(tot & 0xFFFFF);
      const int cnt0 = static_cast<int>(tot >> 32 & 0xFFFFF);
      if (prm.prof != 0 && t == 0 && my_children > LL_CAP) ++sm.prof_wide;
      {
        uint16_t* it = sm.item + (static_cast<int>((woff + incl) & 0xFFFFF) - mine);
#pragma unroll
        for (int q = 0; q < LL_PPT; q++) {
          uint32_t m = cm[q];
          while (m) {
            const int s = __ffs(m) - 1;
            m &= m - 1;
            *it++ = static_cast<uint16_t>(((LL_PPT * t + q) << 5) | s);
          }
        }
      }
      ll_wait(bar_w, T);  // items complete
      TSB_PROF(prof_w, 0, LL_PROF_SCAN)
      // ---- (5) my children (first window), built and evaluated while the other CTAs' counts are on their way
      auto build_window = [&](int c0, int cnt) {
        for (int c = t; c < cnt; c += T)
          sm.stage[c] = ll_build_child<N, REC>(sm.parent, sm.diag, sm.item[c0 + c], &sm.stage_diag[c]);
      };
      build_window(0, min(LL_CAP, my_children));
      TSB_PROF(prof_w, 0, LL_PROF_BUILD)
      // ---- the handoff: my offsets from the exchange warp (also: the first window is complete)
      if (ll_bar_or(bar_hand, TX, false)) break;  // (an abort of the gather)
      TSB_PROF(prof_w, 0, LL_PROF_HAND)
      const int off0 = sm.plan.off0, off1 = sm.plan.off1;

      // ---- (7) my children, in place, tagged with this round's tag (every slice of the chunk has been read: all
      // 2G slots carried this round's epoch)
      for (int c0 = 0; c0 < my_children; c0 += LL_CAP) {
        const int cnt = min(LL_CAP, my_children - c0);
        if (c0 > 0) {
          ll_wait(bar_w, T);  // the previous window has been copied out
          build_window(c0, cnt);
          ll_wait(bar_w, T);
        }
        // child c of my share goes to position s0 + off0 + c (bottom sub-slice) or s0 + off1 + (c - cnt0) (top one)
        unsigned long long* const dst0 = fat[s0 + off0 + c0].w;
        unsigned long long* const dst1 = fat[s0 + off1 + c0 - cnt0].w;
        const int npc = 2 * cnt;  // 16-byte pieces, consecutive lanes on consecutive pieces, four in flight per thread
        for (int pc = t; pc < npc; pc += 4 * T) {
          uint2 d[4];
          uint32_t dm[4];
#pragma unroll
          for (int u = 0; u < 4; u++) {
            const int x = min(pc + u * T, npc - 1);
            d[u] = reinterpret_cast<const uint2*>(sm.stage)[x];
            dm[u] = reinterpret_cast<const uint32_t*>(sm.stage_diag)[x];  // ld or rd
          }
#pragma unroll
          for (int u = 0; u < 4; u++) {
            const int x = pc + u * T;
            unsigned long long a, b;
            ll_piece(d[u].x, d[u].y, dm[u], round_tag, a, b);
            if (x < npc) st_fat2((c0 + (x >> 1) < cnt0 ? dst0 : dst1) + 2 * x, a, b);
          }
        }
      }
      TSB_PROF(prof_w, 0, LL_PROF_STORE)
      // (straight into the next round: sm.plan holds its geometry since the handoff.  No worker barrier is needed
      // before the next poll overwrites sm.parent and sm.diag: every build of this round ended before a barrier all
      // workers passed, and sm.stage and sm.stage_diag are next written after the next poll's barrier, when every
      // store has read them.)
    }
    if (prm.prof != 0) atomicAdd(&sm.prof_fertile, prof_fertile);
  }
  ll_bar_or(bar_hand, TX, false);  // (all threads of the half leave the loop at the same round; the profile is complete)
  if (prm.prof != 0 && t == T) {
    prm.state->cta_fertile[k] = sm.prof_fertile;
    prm.state->cta_wide[k] = sm.prof_wide;
  }
  if (k == 0 && t == T) {
    RoundsState* st = prm.state;
    st->size = size;
    st->size_hi = size_hi;
    st->epoch = epoch;
    st->rounds = rounds;
    st->parents = tot_parents;
    st->children = tot_children;
    st->solutions = tot_solutions;
    st->exit_code = exit_code;
    if (prof_x)
      for (int i = 0; i < LL_PROF_N; i++) st->prof[i] = sm.prof[i];
  }
#undef TSB_PROF
}
template <int N, int T, int MINB, int PPT, int HALVES = 1>
__global__ void __launch_bounds__(HALVES * (T + 32), MINB) nq_rounds_ll_kernel(const __grid_constant__ LlMultiParams mprm) {
  static_assert(HALVES == 1 || (HALVES == 2 && MINB == 1), "two pools per CTA: one CTA per SM");
  nq_rounds_ll_body<N, T, PPT, HALVES, NQ_REC>(mprm);
}
// 25-byte records (wide handles, N <= 24): one pool per launch, one CTA per SM, two parents per worker thread
template <int N>
__global__ void __launch_bounds__(LL_T + 32, 1) nq_rounds_ll_wide_kernel(const __grid_constant__ LlMultiParams mprm) {
  nq_rounds_ll_body<N, LL_T, 2, 1, NQ_REC24>(mprm);
}

// ---- diagnostics (tsb_debug_flag_exchange, tools/flag_exchange.py): cycles per round of bare all-to-all flag exchanges
// among co-resident CTAs, with no evaluation and no children — the floor that ordering the rounds puts under a round,
// and how it scales with the number of CTAs (nq_ll_grid's CTA counts rest on it).  By default a round is two
// exchanges: every CTA publishes a slot and polls all G slots, then releases a "done" flag (st.release) and polls all
// G done flags followed by an acquire fence.  variant bits: 1 = no release fence (plain store of the done flag); 2 = no
// acquire fence; 4 = every thread stores 16 bytes to global before the release (a round's children); 8 = polls are
// weak L2 loads (ld.global.cg) instead of ld.relaxed.gpu; 16 = only ONE exchange per round (the slots); 32 = one
// exchange through per-reader inboxes (every writer stores its flag into every reader's own row)
struct RoundsSync {  // zeroed before the launch
  unsigned long long slot[LL_MAX_SMS];  // 32-bit slots by round parity
  unsigned done[LL_MAX_SMS];            // epoch of the last round this CTA has finished
  unsigned abort;
};
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
template <bool CG>
__device__ __forceinline__ void bench_ld4(const unsigned* p, unsigned& v0, unsigned& v1, unsigned& v2, unsigned& v3) {
  if constexpr (CG)
    asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3) : "l"(p) : "memory");
  else
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3) : "l"(p) : "memory");
}
// warp 0: all G 32-bit flags equal `want`
template <bool CG>
__device__ __forceinline__ bool bench_wait32(const unsigned* f, int G, unsigned want, unsigned* abort_flag) {
  const int lane = threadIdx.x & 31;
  SpinGuard guard;
  for (;;) {
    bool ok = true;
    for (int i = 4 * lane; i < G; i += 128) {
      unsigned v0, v1, v2, v3;
      bench_ld4<CG>(f + i, v0, v1, v2, v3);
      ok &= v0 == want && (i + 1 >= G || v1 == want) && (i + 2 >= G || v2 == want) && (i + 3 >= G || v3 == want);
    }
    if (__all_sync(0xFFFFFFFFu, ok)) return true;
    if (__any_sync(0xFFFFFFFFu, guard.expired(abort_flag))) return false;
  }
}
template <bool CG>
__device__ __forceinline__ void rounds_sync_bench_body(RoundsSync* sy, unsigned epoch0, int rounds, int variant,
                                                       uint4* scratch, long long* out_cycles) {
  const int t = threadIdx.x, wid = t >> 5, k = blockIdx.x, G = gridDim.x;
  unsigned* const slot32 = reinterpret_cast<unsigned*>(sy->slot);  // 32-bit slots: 592 B = 5 lines per sweep
  unsigned epoch = epoch0;
  const long long c0 = clock64();
  for (int r = 0; r < rounds; r++) {
    ++epoch;
    bool ok = true;
    if (!(variant & 16)) {
      if (r > 0 && wid == 0) {
        ok = bench_wait32<CG>(sy->done, G, epoch - 1u, &sy->abort);
        if (!(variant & 2)) __threadfence();
      }
      if (__syncthreads_or(!ok)) break;
    }
    if (variant & 32) {  // per-reader inboxes: writer k stores its flag into row j of every reader j; a reader polls
                         // only its own row (no line is polled by more than one CTA)
      unsigned* const inbox = reinterpret_cast<unsigned*>(scratch) + (r & 1) * 256 * 256;
      for (int j = t; j < G; j += LL_T)
        asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(&inbox[j * 256 + k]), "r"(epoch) : "memory");
      if (wid == 0) ok = bench_wait32<CG>(inbox + k * 256, G, epoch, &sy->abort);
      if (__syncthreads_or(!ok)) break;
      continue;
    }
    unsigned* const sl = slot32 + 256 * (r & 1);  // (two slot arrays, by round parity: a single exchange per round
                                                  // lets a fast CTA publish round r+1 before a slow one has read r)
    if (t == 0) asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(&sl[k]), "r"(epoch) : "memory");
    if (wid == 0) ok = bench_wait32<CG>(sl, G, epoch, &sy->abort);
    if (__syncthreads_or(!ok)) break;
    if (variant & 4) __stcg(scratch + (static_cast<long long>(k) * LL_T + t), make_uint4(epoch, t, k, r));
    if (!(variant & 16)) {
      __syncthreads();
      if (t == 0) {
        if (variant & 1)
          asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(&sy->done[k]), "r"(epoch) : "memory");
        else
          st_release_u32(&sy->done[k], epoch);
      }
    }
  }
  if (k == 0 && t == 0) *out_cycles = clock64() - c0;
}
__global__ void __launch_bounds__(LL_T, 1) rounds_sync_bench_kernel(RoundsSync* sy, unsigned epoch0, int rounds,
                                                                    int variant, uint4* scratch, long long* out_cycles) {
  if (variant & 8)
    rounds_sync_bench_body<true>(sy, epoch0, rounds, variant, scratch, out_cycles);
  else
    rounds_sync_bench_body<false>(sy, epoch0, rounds, variant, scratch, out_cycles);
}

}  // namespace tsb

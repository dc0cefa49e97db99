// tsb_host.cpp — host side of libtsb200: the CPU logic the reference keeps in Chapel, restated in
// C++ only because no Chapel compiler exists on the build / bench hosts (SURVEY.md fact 1):
//   * Taillard instance generator and PFSP table precompute (lib/pfsp/Taillard.chpl,
//     fill_* in lib/pfsp/Bound_simple.chpl / Bound_johnson.chpl) -> tsb_pfsp_tables_build
//   * the 3-step search drivers (nqueens_gpu_chpl.chpl, nqueens_multigpu_chpl.chpl,
//     pfsp_gpu_chpl.chpl, pfsp_multigpu_chpl.chpl) with the same Pool contract
//     (lib/commons/Pool.chpl) and the same --m / --M / --D meaning -> tsb_nq_search, tsb_pfsp_search
// The offload step of those drivers calls tsb_*_evaluate, i.e. exactly the C ABI a patched Chapel
// driver would call (INTEGRATION.md).  Nothing here touches the GPU directly and nothing here
// uses oracle/.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <thread>
#include <type_traits>
#include <vector>

#include "ll_tiers.h"
#include "pfsp_search_pool.h"
#include "search_ckpt.h"
#include "tsb200.h"

namespace {

// ---- Taillard benchmark data (seeds and best-known makespans of ta001..ta120, Taillard 1993;
// the values the reference tabulates in lib/pfsp/Taillard.chpl:3-27, :56-67) ----
const int64_t kSeeds[120] = {
    873654221,  379008056,  1866992158, 216771124,  495070989,  402959317,  1369363414, 2021925980,
    573109518,  88325120,   587595453,  1401007982, 873136276,  268827376,  1634173168, 691823909,
    73807235,   1273398721, 2065119309, 1672900551, 479340445,  268827376,  1958948863, 918272953,
    555010963,  2010851491, 1519833303, 1748670931, 1923497586, 1829909967, 1328042058, 200382020,
    496319842,  1203030903, 1730708564, 450926852,  1303135678, 1273398721, 587288402,  248421594,
    1958948863, 575633267,  655816003,  1977864101, 93805469,   1803345551, 49612559,   1899802599,
    2013025619, 578962478,  1539989115, 691823909,  655816003,  1315102446, 1949668355, 1923497586,
    1805594913, 1861070898, 715643788,  464843328,  896678084,  1179439976, 1122278347, 416756875,
    267829958,  1835213917, 1328833962, 1418570761, 161033112,  304212574,  1539989115, 655816003,
    960914243,  1915696806, 2013025619, 1168140026, 1923497586, 167698528,  1528387973, 993794175,
    450926852,  1462772409, 1021685265, 83696007,   508154254,  1861070898, 26482542,   444956424,
    2115448041, 118254244,  471503978,  1215892992, 135346136,  1602504050, 160037322,  551454346,
    519485142,  383947510,  1968171878, 540872513,  2013025619, 475051709,  914834335,  810642687,
    1019331795, 2056065863, 1342855162, 1325809384, 1988803007, 765656702,  1368624604, 450181436,
    1927888393, 1759567256, 606425239,  19268348,   1298201670, 2041736264, 379756761,  28837162};
const int32_t kBestUb[120] = {
    1278,  1359,  1081,  1293,  1235,  1195,  1234,  1206,  1230,  1108,  1582,  1659,  1496,  1377,  1419,
    1397,  1484,  1538,  1593,  1591,  2297,  2099,  2326,  2223,  2291,  2226,  2273,  2200,  2237,  2178,
    2724,  2834,  2621,  2751,  2863,  2829,  2725,  2683,  2552,  2782,  2991,  2867,  2839,  3063,  2976,
    3006,  3093,  3037,  2897,  3065,  3846,  3699,  3640,  3719,  3610,  3679,  3704,  3691,  3741,  3755,
    5493,  5268,  5175,  5014,  5250,  5135,  5246,  5094,  5448,  5322,  5770,  5349,  5676,  5781,  5467,
    5303,  5595,  5617,  5871,  5845,  6173,  6183,  6252,  6254,  6285,  6331,  6223,  6372,  6247,  6404,
    10862, 10480, 10922, 10889, 10524, 10329, 10854, 10730, 10438, 10675, 11158, 11160, 11281, 11275, 11259,
    11176, 11337, 11301, 11146, 11284, 26040, 26500, 26371, 26456, 26334, 26469, 26389, 26560, 26005, 26457};

double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// growable deque with the reference pool's interface (lib/commons/Pool.chpl:12-73)
template <class Node>
struct Pool {
  std::vector<Node> el;
  size_t front = 0, size = 0;
  Pool() { el.resize(1024); }
  void pushBack(const Node& n) {
    if (front + size >= el.size()) el.resize(el.size() * 2);
    el[front + size] = n;
    ++size;
  }
  bool popBack(Node& n) {
    if (!size) return false;
    n = el[front + --size];
    return true;
  }
  bool popFront(Node& n) {
    if (!size) return false;
    n = el[front++];
    --size;
    return true;
  }
  // Pool.chpl:50-59: nothing below m; otherwise the newest min(size, M) nodes, order preserved
  int popBackBulk(int m, int M, Node* parents) {
    if (size < static_cast<size_t>(m)) return 0;
    const size_t n = std::min(size, static_cast<size_t>(M));
    size -= n;
    std::memcpy(parents, &el[front + size], n * sizeof(Node));
    return static_cast<int>(n);
  }
};

// ------------------------------------------------------------------ N-Queens CPU twin
// Node: tsb_nq_node (N <= 20, tsb_nq_create handles) or tsb_nq_node24 (a MAX_QUEENS = 24 build, tsb_nq_create_wide)
template <class Node>
int nq_create_for(tsb_nq** h, int device, int N, int g, int M) {
  if constexpr (std::is_same_v<Node, tsb_nq_node24>)
    return tsb_nq_create_wide(h, device, TSB_MAX_QUEENS_WIDE, N, g, M);
  else
    return tsb_nq_create(h, device, N, g, M);
}
// isSafe / decompose of the drivers' CPU steps 1 and 3 (nqueens_gpu_chpl.chpl:51-89)
template <class Node>
inline bool nq_safe(const Node& p, int depth, int row_pos) {
  for (int i = 0; i < depth; i++) {
    const int d = depth - i, o = p.board[i];
    if (o == row_pos - d || o == row_pos + d) return false;
  }
  return true;
}
template <class Node>
void nq_decompose(int N, const Node& parent, uint64_t& tree, uint64_t& sol, Pool<Node>& pool) {
  const int depth = parent.depth;
  if (depth == N) {
    ++sol;
    return;
  }
  for (int j = depth; j < N; j++)
    if (nq_safe(parent, depth, parent.board[j])) {
      Node c = parent;
      c.depth = static_cast<uint8_t>(depth + 1);
      std::swap(c.board[depth], c.board[j]);
      pool.pushBack(c);
      ++tree;
    }
}
// nqueens_gpu_chpl.chpl:126-149
template <class Node>
void nq_generate_children(int N, const Node* parents, int size, const uint8_t* labels, uint64_t& tree, uint64_t& sol,
                          Pool<Node>& pool) {
  for (int i = 0; i < size; i++) {
    const Node& parent = parents[i];
    const int depth = parent.depth;
    if (depth == N) {
      ++sol;
      continue;
    }
    const uint8_t* lab = labels + static_cast<size_t>(i) * N;
    for (int j = depth; j < N; j++)
      if (lab[j] == 1) {
        Node c = parent;
        c.depth = static_cast<uint8_t>(depth + 1);
        std::swap(c.board[depth], c.board[j]);
        pool.pushBack(c);
        ++tree;
      }
  }
}

// tsb_search_request_stop: set from any thread or a signal handler, cleared by the search that stops on it
std::atomic<int> g_stop_request{0};
static_assert(std::atomic<int>::is_always_lock_free, "tsb_search_request_stop must be async-signal-safe");

// The stop condition of a resumable search (tsb_*_search[_device]_ckpt): its deadline or a stop request.  A task asks
// between two library calls (device pools) or two offloads (host pools), after its first one; once one task sees it,
// every task stops at its next boundary.
struct StopCtl {
  double deadline = 0;                // now_s() + seconds at the call (infinity: no time limit)
  std::atomic<bool> stopping{false};  // latched
  bool check() {
    if (!stopping.load() && (g_stop_request.load() != 0 || now_s() >= deadline)) stopping.store(true);
    return stopping.load();
  }
};

struct GpuTaskResult {
  uint64_t tree = 0, sol = 0, offloads = 0, parents = 0, launches = 0;
  int64_t best = 0;
  int rc = 0;
  double t_pool_calls = 0;  // seconds inside the library's device-pool calls (TSB200_TRACE)
};

inline void bind_task(int device) {  // one host thread per GPU: next to its GPU (env TSB200_NO_NUMA=1: no)
  if (!std::getenv("TSB200_NO_NUMA")) (void)tsb_bind_thread_to_device(device);
}

// ---- intra-node work stealing between the tasks' DEVICE pools (the reference steals between its per-GPU host
// pools: nqueens_multigpu_chpl.chpl:255-312, pfsp_multigpu_chpl.chpl:438-495).  A task that runs out of work
// (pool below m) asks the task with the fullest pool; the victim serves the request between two of its launches
// (its pool is on its GPU and only it may touch it while kernels run): the oldest half of its pool moves to the
// thief's GPU peer-to-peer (tsb_*_pool_steal = popFrontBulkFree, Pool_par.chpl:178-191).  Termination: all tasks
// idle (util.chpl:16-30).  Counts are split-invariant for N-Queens and for PFSP with --ub 1, so stealing changes
// the per-GPU shares, never the totals.
struct StealBoard {
  explicit StealBoard(int D_) : D(D_), size(D_, 0), request(D_, -1), reply(D_, 0), handle(D_, nullptr), failed(false) {}
  const int D;
  std::mutex mu;
  std::condition_variable cv;
  std::vector<long long> size;  // pool size every task last published
  std::vector<int> request;     // request[v] = thief waiting for victim v, or -1
  std::vector<int> reply;       // reply[thief]: 0 pending, 1 granted, -1 denied
  std::vector<void*> handle;    // the tasks' library handles
  bool failed;                  // a task could not create its handle: nobody steals
  int idle = 0;
  bool done = false;
  bool stop = false;  // a task stopped for a checkpoint: nobody steals, every waiting task stops too
  uint64_t steals = 0;
  // every task's handle exists before anybody steals
  void publish_handle(int me, void* h, long long my_size) {
    std::unique_lock<std::mutex> lk(mu);
    handle[me] = h;
    size[me] = my_size;
    if (!h) failed = true;
    cv.notify_all();
    cv.wait(lk, [&] {
      if (failed) return true;
      for (void* x : handle)
        if (!x) return false;
      return true;
    });
  }
};

// what a device-pool task does between two launches: publish its pool size, serve a pending steal request
// smallest pool worth stealing from: the reference's 2 m (Pool_par.chpl:178-191) for the small chunks of the
// persistent kernel; with large chunks a pool below 2 M is one or two bandwidth-bound rounds of work — splitting
// it costs more (arena reservation on the thief, under-filled launches on both) than it saves (multi-GPU searches
// at M = 4 Mi ran several times slower when every idle task stole half of such pools)
// Small chunks = what one pool's persistent kernel takes on the node's GPUs (device 0's SM count: one model per node).
inline bool small_chunks(int M) {
  return M <= tsb::ll_pool_capacity(tsb_device_sm_count(0), 1);
}
inline long long steal_floor(int m, int M) { return small_chunks(M) ? 2LL * m : std::max<long long>(2LL * m, 2LL * M); }

template <class StealFn>
int board_service(StealBoard* sb, int me, long long my_size, long long floor_, StealFn&& steal) {
  if (!sb) return TSB_OK;
  int thief = -1;
  {
    std::lock_guard<std::mutex> lk(sb->mu);
    sb->size[me] = my_size;
    thief = sb->request[me];
    sb->request[me] = -1;
  }
  if (thief < 0) return TSB_OK;
  int64_t got = 0;
  int rc = TSB_OK;
  if (my_size >= floor_ && !sb->failed) rc = steal(sb->handle[me], sb->handle[thief], &got);
  {
    std::lock_guard<std::mutex> lk(sb->mu);
    sb->reply[thief] = (rc == TSB_OK && got > 0) ? 1 : -1;
    sb->size[me] = my_size - got;
    if (got > 0) ++sb->steals;
  }
  sb->cv.notify_all();
  return rc;
}
// out of work: 1 = stole something (keep going), 0 = everybody is idle (terminate), -1 = the search stops
inline int board_acquire(StealBoard* sb, int me, long long my_size, long long floor_) {
  if (!sb) return 0;
  std::unique_lock<std::mutex> lk(sb->mu);
  sb->size[me] = my_size;
  const auto deny_mine = [&] {  // I have nothing to give
    if (sb->request[me] >= 0) {
      sb->reply[sb->request[me]] = -1;
      sb->request[me] = -1;
      sb->cv.notify_all();
    }
  };
  deny_mine();
  ++sb->idle;
  for (;;) {
    if (sb->stop) {
      deny_mine();
      return -1;
    }
    if (sb->idle == sb->D) {
      sb->done = true;
      sb->cv.notify_all();
      return 0;
    }
    if (sb->done) return 0;
    int v = -1;
    for (int i = 0; i < sb->D && !sb->failed; i++)  // the fullest pool nobody is already asking
      if (i != me && sb->request[i] < 0 && sb->size[i] >= floor_ && (v < 0 || sb->size[i] > sb->size[v])) v = i;
    if (v < 0) {
      deny_mine();
      sb->cv.wait_for(lk, std::chrono::microseconds(200));
      continue;
    }
    sb->request[v] = me;
    sb->reply[me] = 0;
    --sb->idle;  // waiting for a victim is not being idle: the victim may hand over half of its pool
    sb->cv.wait(lk, [&] { return sb->reply[me] != 0 || sb->done; });
    if (sb->reply[me] > 0) return 1;
    if (sb->done) return 0;
    ++sb->idle;
    sb->size[v] = std::min<long long>(sb->size[v], floor_ - 1);  // (it publishes again after its next launch)
  }
}

// a task leaves on an error: nobody may wait for it any more
inline void board_abort(StealBoard* sb, int me) {
  if (!sb) return;
  std::lock_guard<std::mutex> lk(sb->mu);
  sb->failed = sb->done = true;
  if (sb->request[me] >= 0) sb->reply[sb->request[me]] = -1;
  sb->request[me] = -1;
  sb->cv.notify_all();
}

// a task stops for a checkpoint: the request waiting for it is denied, and no task asks anybody any more
inline void board_stop(StealBoard* sb, int me) {
  if (!sb) return;
  std::lock_guard<std::mutex> lk(sb->mu);
  sb->stop = true;
  if (sb->request[me] >= 0) sb->reply[sb->request[me]] = -1;
  sb->request[me] = -1;
  sb->cv.notify_all();
}

// static strided split of the warm-up pool (nqueens_multigpu_chpl.chpl:199-226)
template <class Node>
void static_split(Pool<Node>& pool, int D, std::vector<Pool<Node>>& multi) {
  const size_t poolSize = pool.size, c = poolSize / D, l = poolSize - (D - 1) * c, f = pool.front;
  multi.resize(D);
  for (int g = 0; g < D; g++) {
    for (size_t i = 0; i < c; i++) multi[g].pushBack(pool.el[g + f + i * D]);
    if (g == D - 1)
      for (size_t i = 0; i < l - c; i++) multi[g].pushBack(pool.el[D * c + f + i]);
  }
  pool.front = 0;
  pool.size = 0;
}

// rounds per library call when nodes may move between pools (a victim serves requests between calls)
inline int64_t rounds_per_call(bool moves, int M) { return !moves ? INT64_MAX : small_chunks(M) ? 256 : 4; }

// rounds per call of a resumable search where the search above makes one unbounded call: a stop waits for the call
// in flight, and pool_run resumes bit-exactly, so the cap changes no chunk sequence
constexpr int64_t kCkptRoundsPerCall = 1024;
// (env TSB200_CKPT_ROUNDS overrides that cap, so that tests can stop a search after a few rounds of large chunks)
inline int64_t ckpt_rounds_per_call() {
  const char* v = std::getenv("TSB200_CKPT_ROUNDS");
  return v && std::atoll(v) > 0 ? std::atoll(v) : kCkptRoundsPerCall;
}

// (env set: nodes never move between the device pools of a search, the static split alone)
inline bool steal_allowed() { return !std::getenv("TSB200_NO_STEAL"); }

// ---- the device pools of one task, for either handle type: the library's pool calls, overloaded on the handle
inline int64_t pool_size(const tsb_nq* h) { return tsb_nq_pool_size(h); }
inline int64_t pool_size(const tsb_pfsp* h) { return tsb_pfsp_pool_size(h); }
inline int pool_push(tsb_nq* h, const void* nodes, int64_t n) { return tsb_nq_pool_push(h, nodes, n); }
inline int pool_push(tsb_pfsp* h, const void* nodes, int64_t n) { return tsb::search::pfsp_pool_push(h, nodes, n); }
inline int pool_drain(tsb_nq* h, void* nodes, int64_t cap, int64_t* n) { return tsb_nq_pool_drain(h, nodes, cap, n); }
inline int pool_drain(tsb_pfsp* h, void* nodes, int64_t cap, int64_t* n) { return tsb_pfsp_pool_drain(h, nodes, cap, n); }
inline int pool_steal(tsb_nq* v, tsb_nq* t, int m, int64_t* got) { return tsb_nq_pool_steal(v, t, m, got); }
inline int pool_steal(tsb_pfsp* v, tsb_pfsp* t, int m, int64_t* got) { return tsb_pfsp_pool_steal(v, t, m, got); }
inline int pool_sibling(tsb_nq* h, int i, tsb_nq** sib) { return tsb_nq_sibling(h, i, sib); }
inline int pool_sibling(tsb_pfsp* h, int i, tsb_pfsp** sib) { return tsb::search::pfsp_sibling(h, i, sib); }
inline uint64_t kernel_launches(const tsb_nq* h) { return tsb_nq_kernel_launches(h); }
inline uint64_t kernel_launches(const tsb_pfsp* h) { return tsb_pfsp_kernel_launches(h); }

// drain a device pool and push what it held onto a host pool
template <class H, class Node>
int drain_to_host(H* h, Pool<Node>& pool) {
  const int64_t left = pool_size(h);
  std::vector<Node> rest(static_cast<size_t>(left) + 1);
  int64_t n = 0;
  const int rc = pool_drain(h, rest.data(), left, &n);
  for (int64_t i = 0; i < n && rc == TSB_OK; i++) pool.pushBack(rest[i]);
  return rc;
}
// drain a device pool into records of `rec` bytes, in logical order
template <class H>
int drain_to_bytes(H* h, size_t rec, std::vector<uint8_t>& out) {
  const int64_t left = pool_size(h);
  std::vector<uint8_t> buf((static_cast<size_t>(left) + 1) * rec);
  int64_t n = 0;
  const int rc = pool_drain(h, buf.data(), left, &n);
  buf.erase(buf.begin() + static_cast<long>(rc == TSB_OK ? static_cast<size_t>(n) * rec : 0), buf.end());
  out.swap(buf);
  return rc;
}

// one task's share of a resumable search: the pools it resumes from (nullptr: it starts from its share of step 1; a
// host-pool task has exactly one), the search's stop condition, and, when it stopped, the pools it left
struct TaskCkpt {
  const std::vector<tsb::ckpt::PoolState>* resume = nullptr;
  StopCtl* stop = nullptr;
  bool stopped = false;
  std::vector<tsb::ckpt::PoolState> pools;
};

// a host pool's nodes, front to back, as records of a checkpoint, and back
template <class Node>
std::vector<uint8_t> pool_records(const Pool<Node>& pool) {
  const auto* b = reinterpret_cast<const uint8_t*>(pool.el.data() + pool.front);
  return std::vector<uint8_t>(b, b + pool.size * sizeof(Node));
}
template <class Node>
void push_records(const std::vector<uint8_t>& rec, Pool<Node>& pool) {
  for (size_t i = 0; i + sizeof(Node) <= rec.size(); i += sizeof(Node)) {
    Node n;
    std::memcpy(&n, &rec[i], sizeof(Node));
    pool.pushBack(n);
  }
}

// The offload loop of one host-pool task (the drivers' step 2: nqueens_gpu_chpl.chpl:197-215, pfsp_gpu_chpl.chpl:
// 373-395): popBackBulk(m, M), `offload` the chunk (one library call: evaluate, then generate_children on the host),
// until the pool holds fewer than m nodes.  `ck` (a resumable search): the task resumes its pool and incumbent from
// the checkpoint, and asks for a stop after every offload, never before its first one; when it stops it leaves its
// pool, front to back, and its incumbent in ck->pools.  A host task never steals, so the chunk sequence across stops
// is the uninterrupted one.
template <class Node, class Offload>
void host_pool_loop(int m, int M, Pool<Node>& pool, Node* parents, GpuTaskResult& r, TaskCkpt* ck, Offload&& offload) {
  if (ck && ck->resume) {
    const tsb::ckpt::PoolState& in = ck->resume->front();  // (load: exactly one per unfinished host task)
    push_records(in.nodes, pool);
    r.best = in.best;
  }
  for (;;) {
    const int n = pool.popBackBulk(m, M, parents);
    if (n <= 0) break;
    r.rc = offload(n);
    if (r.rc != TSB_OK) break;
    ++r.offloads;
    r.parents += static_cast<uint64_t>(n);
    if (ck && ck->stop->check()) {
      ck->stopped = true;
      ck->pools.assign(1, tsb::ckpt::PoolState{r.best, pool_records(pool)});
      break;
    }
  }
}

// The offload loop of one task whose P >= 1 pools (a handle and its siblings) are resident on the device: all rounds
// of step 2 inside the library (one persistent kernel for small M, two kernels per round otherwise; the pools' rounds
// share its launches, S::run_multi = tsb_*_pool_run_multi), `rounds` rounds per call; the host only reads counters.
// `balance`: a pool of the group that runs dry takes the oldest half of the fullest one (as between tasks).  Between
// two calls a thief task is served from the fullest pool of the group.  best[i]: pool i's incumbent.  `stop` (a
// resumable search): asked after every call; true = the task stopped with its pools as they are.
template <class S, class H>
bool devpool_rounds(const S& s, const std::vector<H*>& hs, int m, int M, int64_t rounds, bool balance, StealBoard* sb,
                    int me, int64_t* best, GpuTaskResult& r, StopCtl* stop) {
  const int P = static_cast<int>(hs.size());
  const auto fullest = [&] {
    int v = 0;
    for (int i = 1; i < P; i++)
      if (pool_size(hs[i]) > pool_size(hs[v])) v = i;
    return v;
  };
  const auto steal = [&](void*, void* t, int64_t* got) { return pool_steal(hs[fullest()], static_cast<H*>(t), m, got); };
  const long long floor_ = steal_floor(m, M);
  std::vector<uint64_t> out(4 * P);
  while (r.rc == TSB_OK) {
    if (balance) {
      for (int i = 0; i < P && r.rc == TSB_OK; i++) {
        if (pool_size(hs[i]) >= m) continue;
        const int v = fullest();
        if (v == i || pool_size(hs[v]) < floor_) break;
        int64_t got = 0;
        r.rc = pool_steal(hs[v], hs[i], m, &got);
      }
      if (r.rc != TSB_OK) break;
    }
    long long most = 0, total = 0;
    for (H* x : hs) {
      most = std::max<long long>(most, pool_size(x));
      total += pool_size(x);
    }
    if (most < m) {
      const int got = board_acquire(sb, me, total, floor_);
      if (got < 0) return true;
      if (got == 0) break;
      continue;
    }
    const double c0 = now_s();
    r.rc = s.run_multi(hs.data(), P, m, M, rounds, best, out.data());
    r.t_pool_calls += now_s() - c0;
    if (r.rc != TSB_OK) break;
    for (int i = 0; i < P; i++) {
      r.offloads += out[4 * i];
      r.parents += out[4 * i + 1];
      r.tree += out[4 * i + 2];
      r.sol += out[4 * i + 3];
    }
    r.rc = board_service(sb, me, pool_size(hs[fullest()]), floor_, steal);
    if (r.rc == TSB_OK && stop && stop->check()) {
      board_stop(sb, me);
      return true;
    }
  }
  if (r.rc != TSB_OK) board_abort(sb, me);
  return false;
}

// One task's step 2 on device pools: its pool -> the P = S::pools_on(h, M) device pools of h and its siblings (for
// P > 1 split once more, by the reference's own strided split), all rounds, and the leftovers (fewer than m nodes per
// pool) back to the task's pool.  Each of several pools is one reference task with its own incumbent
// (pfsp_multigpu_chpl.chpl:384), min-reduced here, and hands its leftovers back as a reference task does (popBack).
// `ck` (a resumable search): the task resumes its pools and incumbents from a checkpoint instead of splitting its pool,
// caps unbounded calls at ckpt_rounds_per_call() rounds, and when it stops leaves its pools in ck->pools.
template <class S, class H, class Node>
void devpool_on(const S& s, H* h, int m, int M, Pool<Node>& pool, GpuTaskResult& r, StealBoard* sb, int me,
                TaskCkpt* ck) {
  const uint64_t l0 = kernel_launches(h);
  const int P = s.pools_on(h, M);
  const std::vector<tsb::ckpt::PoolState>* resume = ck ? ck->resume : nullptr;
  if (resume && static_cast<int>(resume->size()) != P) r.rc = TSB_EINVAL;  // (written where P differed)
  std::vector<H*> hs{h};
  for (int i = 1; i < P && r.rc == TSB_OK; i++) {
    H* sib = nullptr;
    r.rc = pool_sibling(h, i, &sib);
    hs.push_back(sib);
  }
  std::unique_ptr<int64_t[]> best(new int64_t[P]);
  std::fill(best.get(), best.get() + P, r.best);
  long long most = 0;
  if (resume) {
    for (int i = 0; i < P && r.rc == TSB_OK; i++) {
      const tsb::ckpt::PoolState& in = (*resume)[i];
      if (!in.nodes.empty()) r.rc = pool_push(hs[i], in.nodes.data(), static_cast<int64_t>(in.nodes.size() / sizeof(Node)));
      best[i] = in.best;
      most = std::max<long long>(most, pool_size(hs[i]));
    }
  } else {
    std::vector<Pool<Node>> part;
    if (r.rc == TSB_OK) static_split(pool, P, part);
    for (int i = 0; i < P && r.rc == TSB_OK; i++) {
      r.rc = pool_push(hs[i], &part[i].el[part[i].front], static_cast<int64_t>(part[i].size));
      most = std::max<long long>(most, pool_size(hs[i]));
    }
  }
  if (sb) sb->publish_handle(me, r.rc == TSB_OK ? h : nullptr, most);
  int64_t rounds = s.rounds(P, sb != nullptr, M);
  if (ck && rounds == INT64_MAX) rounds = ckpt_rounds_per_call();
  bool stopped = false;
  if (r.rc == TSB_OK)
    stopped = devpool_rounds(s, hs, m, M, rounds, s.balance, sb, me, best.get(), r, ck ? ck->stop : nullptr);
  r.best = *std::min_element(best.get(), best.get() + P);
  if (std::getenv("TSB200_TRACE"))  // (the rounds alone: no handle set-up, pool push or drain)
    std::fprintf(stderr, "[tsb200] task %d: %d pools, %llu rounds in %.3f ms of pool calls\n", me, P,
                 static_cast<unsigned long long>(r.offloads), r.t_pool_calls * 1e3);
  if (stopped) {  // every pool with its incumbent, in logical order, for the checkpoint
    ck->stopped = true;
    ck->pools.resize(P);
    for (int i = 0; i < P && r.rc == TSB_OK; i++) {
      ck->pools[i].best = best[i];
      r.rc = drain_to_bytes(hs[i], sizeof(Node), ck->pools[i].nodes);
    }
  }
  for (H* x : hs) {
    if (r.rc != TSB_OK || stopped) break;
    Pool<Node> rest;
    r.rc = drain_to_host(x, P == 1 ? pool : rest);
    for (Node n; rest.popBack(n);) pool.pushBack(n);
  }
  r.launches += kernel_launches(h) - l0;
}

// Several pools per task (TSB200_POOLS=1 turns it off, =2 caps it at two): for chunks that fit the persistent kernel a
// round is a chain of L2 round trips with little work in between, so the task's share of the warm-up pool is split
// once more — the reference's own strided split (static_split) — into P device pools (P = tsb_nq_pools_per_launch: 4
// on an H100 for M <= 50688) whose rounds run in ONE launch (tsb_nq_pool_run_multi), two CTAs of different pools on
// every SM filling each other's waits.  Each pool follows the reference's rule on its own nodes: for D tasks the
// chunk sequence is that of a 2-level split into P D pools, the totals are split-invariant.
inline int nq_pools_wanted(int M) {  // (decides the warm-up size, before any handle exists)
  int cap = 4;
  if (const char* v = std::getenv("TSB200_POOLS")) cap = std::max(1, std::min(4, std::atoi(v)));
  // the persistent kernel's tiers (ll_tiers.h) on device 0's SM count: the GPUs of one node are one model
  return std::min(cap, tsb::ll_pools_for(tsb_device_sm_count(0), M));
}
inline int nq_pools_of(tsb_nq* h, int M) { return std::min(nq_pools_wanted(M), tsb_nq_pools_per_launch(h, M)); }

// Handles of the device-pool drivers are kept between searches (per device, N, g, M): a handle with its sibling
// pools, arenas and fat arenas is ~1.4 GB of cudaMalloc / cudaFree per GPU, which at 8 GPUs cost more than the N = 17
// search itself.  (The Chapel drivers declare their device arrays once, outside the search loop, as well.)
// At most two idle handles are kept per device; tsb_release_cached_handles frees them all.
// (rec: the node width of the handle, 21 or 25 bytes)
struct NqHandleCache {
  struct Entry {
    int device, N, g, M;
    size_t rec;
    tsb_nq* h;
  };
  std::mutex mu;
  std::vector<Entry> idle;
  template <class Node>
  tsb_nq* acquire(int device, int N, int g, int M, int* rc) {
    {
      std::lock_guard<std::mutex> lk(mu);
      for (size_t i = 0; i < idle.size(); i++)
        if (idle[i].device == device && idle[i].N == N && idle[i].g == g && idle[i].M == M && idle[i].rec == sizeof(Node)) {
          tsb_nq* h = idle[i].h;
          idle.erase(idle.begin() + static_cast<long>(i));
          *rc = TSB_OK;
          return h;
        }
    }
    tsb_nq* h = nullptr;
    *rc = nq_create_for<Node>(&h, device, N, g, M);
    return *rc == TSB_OK ? h : nullptr;
  }
  void release(tsb_nq* h, int device, int N, int g, int M, size_t rec, bool healthy) {
    if (!h) return;
    if (!healthy || std::getenv("TSB200_NO_HANDLE_CACHE")) {
      tsb_nq_destroy(h);
      return;
    }
    // at most two idle handles per device (a handle with four pools holds ~1.4 GB): the oldest one goes
    tsb_nq* evict = nullptr;
    {
      std::lock_guard<std::mutex> lk(mu);
      idle.push_back({device, N, g, M, rec, h});
      int on_device = 0;
      for (const Entry& e : idle) on_device += e.device == device;
      if (on_device > 2)
        for (size_t i = 0; i < idle.size(); i++)
          if (idle[i].device == device) {
            evict = idle[i].h;
            idle.erase(idle.begin() + static_cast<long>(i));
            break;
          }
    }
    if (evict) tsb_nq_destroy(evict);
  }
  void clear() {
    std::lock_guard<std::mutex> lk(mu);
    for (Entry& e : idle) tsb_nq_destroy(e.h);
    idle.clear();
  }
};
NqHandleCache& nq_handle_cache() {
  static NqHandleCache* c = new NqHandleCache();  // (never destroyed: no CUDA calls at process exit)
  return *c;
}

// ------------------------------------------------------------------ PFSP CPU twin
int64_t unif(int64_t& seed, int64_t low, int64_t high) {  // lib/pfsp/Taillard.chpl:72-84
  const int64_t m = 2147483647, a = 16807, b = 127773, c = 2836;
  const int64_t k = seed / b;
  seed = a * (seed % b) - k * c;
  if (seed < 0) seed += m;
  const double v = static_cast<double>(seed) / static_cast<double>(m);
  return low + static_cast<int64_t>(v * static_cast<double>(high - low + 1));
}

// CPU bounds used by decompose in steps 1 and 3 (pfsp_gpu_chpl.chpl:88-189), on the tables of a MAX_JOBS = 20
// (tsb_pfsp_tables) or 50 (tsb_pfsp_tables50) build
template <class Tables>
struct HostBounds {
  static constexpr int kMaxJobs = sizeof(Tables::p_times) / sizeof(int32_t) / TSB_MAX_MACHINES;
  static_assert(kMaxJobs <= 64, "the scheduled set of lb2 is a 64-bit mask");
  const Tables& t;
  explicit HostBounds(const Tables& tt) : t(tt) {}
  void front_of(const int32_t* prmu, int limit1, int32_t* F) const {  // schedule_front
    const int N = t.jobs, M = t.machines;
    if (limit1 == -1) {
      for (int j = 0; j < M; j++) F[j] = t.min_heads[j];
      return;
    }
    std::fill(F, F + M, 0);
    for (int i = 0; i <= limit1; i++) {
      const int job = prmu[i];
      F[0] += t.p_times[job];
      for (int j = 1; j < M; j++) F[j] = std::max(F[j - 1], F[j]) + t.p_times[j * N + job];
    }
  }
  void remain_of(const int32_t* prmu, int limit1, int32_t* R) const {  // sum_unscheduled
    const int N = t.jobs, M = t.machines;
    std::fill(R, R + M, 0);
    for (int k = limit1 + 1; k < N; k++)
      for (int j = 0; j < M; j++) R[j] += t.p_times[j * N + prmu[k]];
  }
  int32_t lb1(const int32_t* prmu, int limit1) const {  // lb1_bound
    const int M = t.machines;
    int32_t F[TSB_MAX_MACHINES], R[TSB_MAX_MACHINES];
    front_of(prmu, limit1, F);
    remain_of(prmu, limit1, R);
    int32_t tmp0 = F[0] + R[0], lb = tmp0 + t.min_tails[0];
    for (int i = 1; i < M; i++) {
      const int32_t tmp1 = std::max(tmp0, F[i] + R[i]);
      lb = std::max(lb, tmp1 + t.min_tails[i]);
      tmp0 = tmp1;
    }
    return lb;
  }
  void lb1_children(const int32_t* prmu, int limit1, int32_t* lb_begin) const {  // lb1_children_bounds
    const int N = t.jobs, M = t.machines;
    int32_t F[TSB_MAX_MACHINES], R[TSB_MAX_MACHINES];
    front_of(prmu, limit1, F);
    remain_of(prmu, limit1, R);
    std::fill(lb_begin, lb_begin + kMaxJobs, 0);
    for (int i = limit1 + 1; i < N; i++) {
      const int job = prmu[i];
      int32_t lb = F[0] + R[0] + t.min_tails[0], tmp0 = F[0] + t.p_times[job];
      for (int k = 1; k < M; k++) {
        const int32_t tmp1 = std::max(tmp0, F[k]);
        lb = std::max(lb, tmp1 + R[k] + t.min_tails[k]);
        tmp0 = tmp1 + t.p_times[k * N + job];
      }
      lb_begin[job] = lb;
    }
  }
  int32_t lb2(const int32_t* prmu, int limit1, int64_t best) const {  // lb2_bound
    const int N = t.jobs;
    int32_t F[TSB_MAX_MACHINES];
    front_of(prmu, limit1, F);
    uint64_t sched = 0;
    for (int j = 0; j <= limit1; j++) sched |= 1ull << prmu[j];
    int32_t lb = 0;
    for (int l = 0; l < t.pairs; l++) {
      const int i = t.mp_order[l], a = t.mp0[i], b = t.mp1[i];
      int32_t t0 = F[a], t1 = F[b];
      for (int j = 0; j < N; j++) {
        const int job = t.johnson[i * N + j];
        if (!((sched >> job) & 1ull)) {
          t0 += t.p_times[a * N + job];
          t1 = std::max(t1, t0 + t.lags[i * N + job]) + t.p_times[b * N + job];
        }
      }
      lb = std::max(lb, std::max(t1 + t.min_tails[b], t0 + t.min_tails[a]));
      if (static_cast<int64_t>(lb) > best) break;
    }
    return lb;
  }
};

template <class Node>
inline void pfsp_child(const Node& parent, int i, Node& c) {
  c = parent;
  c.depth = parent.depth + 1;
  c.limit1 = parent.limit1 + 1;
  std::swap(c.prmu[parent.depth], c.prmu[i]);
}

// decompose (pfsp_gpu_chpl.chpl:88-189)
template <class Tables, class Node>
void pfsp_decompose(const HostBounds<Tables>& hb, int lb_kind, const Node& parent, uint64_t& tree, uint64_t& sol,
                    int64_t& best, Pool<Node>& pool) {
  const int jobs = hb.t.jobs;
  int32_t lb_begin[HostBounds<Tables>::kMaxJobs];
  if (lb_kind == TSB_LB1_D) hb.lb1_children(parent.prmu, parent.limit1, lb_begin);
  for (int i = parent.limit1 + 1; i < jobs; i++) {
    Node c;
    pfsp_child(parent, i, c);
    const int32_t lb = lb_kind == TSB_LB1_D ? lb_begin[parent.prmu[i]]
                       : lb_kind == TSB_LB1 ? hb.lb1(c.prmu, c.limit1)
                                            : hb.lb2(c.prmu, c.limit1, best);
    if (c.depth == jobs) {
      ++sol;
      if (lb < best) best = lb;
    } else if (lb < best) {
      pool.pushBack(c);
      ++tree;
    }
  }
}

// generate_children (pfsp_gpu_chpl.chpl:273-303)
template <class Node>
void pfsp_generate_children(int jobs, const Node* parents, int size, const int32_t* bounds, uint64_t& tree,
                            uint64_t& sol, int64_t& best, Pool<Node>& pool) {
  for (int i = 0; i < size; i++) {
    const Node& parent = parents[i];
    const int depth = parent.depth;
    for (int j = parent.limit1 + 1; j < jobs; j++) {
      const int32_t lb = bounds[j + static_cast<size_t>(i) * jobs];
      if (depth + 1 == jobs) {
        ++sol;
        if (lb < best) best = lb;
      } else if (lb < best) {
        Node c;
        pfsp_child(parent, j, c);
        pool.pushBack(c);
        ++tree;
      }
    }
  }
}

// lbound1 / lbound2 of a Taillard instance (pfsp_gpu_chpl.chpl:325-332) into either table struct
template <class T, int MAXJ>
int build_tables(T* t, int inst, int variant) {
  if (!t || inst < 1 || inst > 120 || variant < 0 || variant > 3) return TSB_EINVAL;
  std::memset(t, 0, sizeof(*t));
  const int N = t->jobs = tsb_taillard_nb_jobs(inst);
  const int M = t->machines = tsb_taillard_nb_machines(inst);
  if (N > MAXJ) return TSB_EUNSUPPORTED;  // MAX_JOBS (lib/pfsp/PFSP_node.chpl:7): 20, or 50 for the wide tables
  int64_t seed = kSeeds[inst - 1];
  for (int i = 0; i < M; i++)  // lib/pfsp/Taillard.chpl:86-97
    for (int j = 0; j < N; j++) t->p_times[i * N + j] = static_cast<int32_t>(unif(seed, 1, 99));
  // fill_min_heads_tails, lib/pfsp/Bound_simple.chpl:254-289.  Chapel's line 271 assigns
  // min(max(int(32)), tmp0): min_heads ends as the head times of the LAST job (SURVEY A.1);
  // the Chapel program is the parity target, so that is what is reproduced here.
  t->min_heads[0] = 0;
  {
    int32_t acc = t->p_times[N - 1];
    for (int k = 1; k < M; k++) {
      t->min_heads[k] = acc;
      acc += t->p_times[k * N + (N - 1)];
    }
  }
  for (int k = 0; k < M; k++) t->min_tails[k] = INT32_MAX;
  t->min_tails[M - 1] = 0;
  for (int i = 0; i < N; i++) {
    int32_t acc = t->p_times[(M - 1) * N + i];
    for (int k = M - 2; k >= 0; k--) {
      t->min_tails[k] = std::min(t->min_tails[k], acc);
      acc += t->p_times[k * N + i];
    }
  }
  // fill_machine_pairs (Bound_johnson.chpl:50-87: LB2_FULL / LB2_LEARN = all pairs, the branch the reference
  // compiles; LB2_NABESHIMA = adjacent machines, LB2_LAGEWEG = each machine with the last) + fill_lags (:89-104)
  int c = 0;
  const auto add_pair = [&](int a, int b) {
    t->mp0[c] = a;
    t->mp1[c] = b;
    t->mp_order[c] = c;
    for (int j = 0; j < N; j++) {
      int32_t s = 0;
      for (int k = a + 1; k < b; k++) s += t->p_times[k * N + j];
      t->lags[c * N + j] = s;
    }
    ++c;
  };
  if (variant == TSB_LB2_NABESHIMA) {
    for (int a = 0; a < M - 1; a++) add_pair(a, a + 1);
  } else if (variant == TSB_LB2_LAGEWEG) {
    for (int a = 0; a < M - 1; a++) add_pair(a, M - 1);
  } else {
    for (int a = 0; a < M - 1; a++)
      for (int b = a + 1; b < M; b++) add_pair(a, b);
  }
  t->pairs = c;
  // fill_johnson_schedules (:145-177): Johnson's rule per pair on (p_a + lag, p_b + lag)
  for (int k = 0; k < t->pairs; k++) {
    const int a = t->mp0[k], b = t->mp1[k];
    int order[MAXJ];
    int32_t k1[MAXJ], k2[MAXJ];
    for (int j = 0; j < N; j++) {
      order[j] = j;
      k1[j] = t->p_times[a * N + j] + t->lags[k * N + j];
      k2[j] = t->p_times[b * N + j] + t->lags[k * N + j];
    }
    std::stable_sort(order, order + N, [&](int x, int y) {
      const bool px = k1[x] < k2[x], py = k1[y] < k2[y];  // partition 0 (k1 < k2) first
      if (px != py) return px;
      return px ? k1[x] < k1[y] : k2[x] > k2[y];
    });
    for (int j = 0; j < N; j++) t->johnson[k * N + j] = order[j];
  }
  return TSB_OK;
}

// ------------------------------------------------------------------ the 3-step search
// The problems of the search.  Each gives the root node and decompose, the incumbent the search starts from (N-Queens:
// 0), the task of one device on its host pool (host_task) or on device pools (device_task), `pools` (device pools per
// task: step 1 warms up D·m·pools nodes), whether device-pool tasks `steal` from each other, and for the device pools
// of one task (devpool_on): how many a handle takes, the rounds per library call, `balance` and run_multi.

// N-Queens on boards of up to 20 queens (tsb_nq_node) or, on wide handles, 24 (tsb_nq_node24)
template <class NodeT>
struct NqSearch {
  using Node = NodeT;
  using Handle = tsb_nq;
  static constexpr bool wide = std::is_same_v<Node, tsb_nq_node24>;
  int N, g;
  bool devpool;
  int pools;  // (one on wide handles, which do not share launches of the persistent kernel)
  bool steal, balance;
  int64_t initial_best = 0;
  NqSearch(int N_, int g_, int M, bool devpool_)
      : N(N_), g(g_), devpool(devpool_), pools(devpool_ && !wide ? nq_pools_wanted(M) : 1),
        steal(devpool_ && steal_allowed()), balance(steal) {}
  Node root() const {
    Node root{};
    for (int i = 0; i < N; i++) root.board[i] = static_cast<uint8_t>(i);
    return root;
  }
  void decompose(const Node& parent, uint64_t& tree, uint64_t& sol, int64_t&, Pool<Node>& pool) const {
    nq_decompose(N, parent, tree, sol, pool);
  }
  // one GPU task's offload loop (nqueens_gpu_chpl.chpl:197-215; nqueens_multigpu_chpl.chpl:234-253)
  void host_task(int device, int m, int M, Pool<Node>& pool, GpuTaskResult& r, TaskCkpt* ck) const {
    tsb_nq* h = nullptr;
    r.rc = nq_create_for<Node>(&h, device, N, g, M);
    if (r.rc != TSB_OK) return;
    std::vector<Node> parents(M);
    std::vector<uint8_t> labels(static_cast<size_t>(M) * N);
    // the chunk arrays live for the whole step 2 (nqueens_gpu_chpl.chpl:191-192): page-lock them once
    tsb_nq_register_host(h, parents.data(), parents.size() * sizeof(Node));
    tsb_nq_register_host(h, labels.data(), labels.size());
    host_pool_loop(m, M, pool, parents.data(), r, ck, [&](int n) {
      const int rc = tsb_nq_evaluate(h, parents.data(), n, labels.data());
      if (rc == TSB_OK) nq_generate_children(N, parents.data(), n, labels.data(), r.tree, r.sol, pool);
      return rc;
    });
    r.launches += tsb_nq_kernel_launches(h);
    tsb_nq_destroy(h);
  }
  void device_task(int device, int m, int M, Pool<Node>& pool, GpuTaskResult& r, StealBoard* sb, int me,
                   TaskCkpt* ck) const {
    const double tt0 = now_s();
    tsb_nq* h = nq_handle_cache().acquire<Node>(device, N, g, M, &r.rc);
    if (r.rc != TSB_OK) {
      if (sb) sb->publish_handle(me, nullptr, 0);
      return;
    }
    const double tt1 = now_s();
    devpool_on(*this, h, m, M, pool, r, sb, me, ck);
    const double tt2 = now_s();
    nq_handle_cache().release(h, device, N, g, M, sizeof(Node), r.rc == TSB_OK);
    if (std::getenv("TSB200_TRACE"))
      std::fprintf(stderr, "[tsb200] device %d: create %.1f ms, %llu rounds in %.1f ms, destroy %.1f ms\n", device,
                   (tt1 - tt0) * 1e3, static_cast<unsigned long long>(r.offloads), (tt2 - tt1) * 1e3,
                   (now_s() - tt2) * 1e3);
  }
  int pools_on(tsb_nq* h, int M) const { return nq_pools_of(h, M); }
  // (with no thief to serve, the dry pools of a group rebalance every 2048 rounds)
  int64_t rounds(int P, bool sb, int M) const { return P == 1 || sb ? rounds_per_call(sb, M) : 2048; }
  int run_multi(tsb_nq* const* hs, int P, int m, int M, int64_t rounds, int64_t*, uint64_t* out) const {
    return tsb_nq_pool_run_multi(hs, P, m, M, rounds, out);
  }
};

// a handle of the build the tables are for: tsb_pfsp_create (20 jobs) or tsb_pfsp_create_wide (50 jobs)
inline int pfsp_create_for(tsb_pfsp** h, int device, int M, const tsb_pfsp_tables* t) {
  return tsb_pfsp_create_from_tables(h, device, M, t);
}
inline int pfsp_create_for(tsb_pfsp** h, int device, int M, const tsb_pfsp_tables50* t) {
  return tsb_pfsp_create50_from_tables(h, device, M, t);
}

// PFSP on the tables of a Taillard instance; `pools` device pools per task, as many as the caller asks for.
// Node / Tables: tsb_pfsp_node / tsb_pfsp_tables (MAX_JOBS = 20) or tsb_pfsp_node50 / tsb_pfsp_tables50 (MAX_JOBS = 50:
// 50-job handles, whose device pools share the launches of their own persistent kernel, pfsp_wide_rounds.cuh)
template <class NodeT, class Tables>
struct PfspSearch {
  using Node = NodeT;
  using Handle = tsb_pfsp;
  HostBounds<Tables> hb;
  int lb_kind;
  bool devpool;
  int pools;
  // moves between pools keep the counts only while best is constant: --ub 1 (SURVEY A.6)
  bool steal, balance;
  int64_t initial_best;
  PfspSearch(const Tables& t, int inst, int lb_kind_, int ub, bool devpool_, int pools_)
      : hb(t), lb_kind(lb_kind_), devpool(devpool_), pools(pools_), steal(devpool_ && ub == 1 && steal_allowed()),
        balance(pools_ > 1 && ub == 1 && steal_allowed()),
        initial_best(ub == 1 ? tsb_taillard_best_ub(inst) : INT64_MAX) {}  // pfsp_gpu_chpl.chpl:37
  Node root() const {
    Node root{};
    root.limit1 = -1;
    for (int i = 0; i < hb.t.jobs; i++) root.prmu[i] = i;
    return root;
  }
  void decompose(const Node& parent, uint64_t& tree, uint64_t& sol, int64_t& best, Pool<Node>& pool) const {
    pfsp_decompose(hb, lb_kind, parent, tree, sol, best, pool);
  }
  void host_task(int device, int m, int M, Pool<Node>& pool, GpuTaskResult& r, TaskCkpt* ck) const {
    tsb_pfsp* h = nullptr;
    r.rc = pfsp_create_for(&h, device, M, &hb.t);
    if (r.rc != TSB_OK) return;
    const int jobs = hb.t.jobs;
    std::vector<Node> parents(M);
    std::vector<int32_t> bounds(static_cast<size_t>(M) * jobs);
    // the chunk arrays live for the whole step 2 (pfsp_gpu_chpl.chpl:355-356): page-lock them once
    tsb_pfsp_register_host(h, parents.data(), parents.size() * sizeof(Node));
    tsb_pfsp_register_host(h, bounds.data(), bounds.size() * sizeof(int32_t));
    host_pool_loop(m, M, pool, parents.data(), r, ck, [&](int n) {
      const int rc = tsb_pfsp_evaluate(h, lb_kind, parents.data(), n, r.best, bounds.data());
      if (rc == TSB_OK) pfsp_generate_children(jobs, parents.data(), n, bounds.data(), r.tree, r.sol, r.best, pool);
      return rc;
    });
    r.launches += tsb_pfsp_kernel_launches(h);
    tsb_pfsp_destroy(h);
  }
  void device_task(int device, int m, int M, Pool<Node>& pool, GpuTaskResult& r, StealBoard* sb, int me,
                   TaskCkpt* ck) const {
    tsb_pfsp* h = nullptr;
    r.rc = pfsp_create_for(&h, device, M, &hb.t);
    if (r.rc != TSB_OK) {
      if (sb) sb->publish_handle(me, nullptr, 0);
      return;
    }
    devpool_on(*this, h, m, M, pool, r, sb, me, ck);
    tsb_pfsp_destroy(h);
  }
  int pools_on(tsb_pfsp*, int) const { return pools; }
  int64_t rounds(int, bool sb, int M) const { return rounds_per_call(balance || sb, M); }
  int run_multi(tsb_pfsp* const* hs, int P, int m, int M, int64_t rounds, int64_t* best, uint64_t* out) const {
    return tsb::search::pfsp_pool_run_multi(hs, P, lb_kind, m, M, rounds, best, out);
  }
};

// A resumable search (tsb_*_search_device_ckpt): where its checkpoint goes and with which parameters, the state it
// resumes from (nullptr: a new search) and its stop condition
struct SearchCkpt {
  const char* path;
  tsb::ckpt::Params params;
  const tsb::ckpt::State* resume;
  StopCtl stop;
};

// The drivers' search (nqueens_multigpu_chpl.chpl, pfsp_multigpu_chpl.chpl; D = 1: nqueens_gpu_chpl.chpl,
// pfsp_gpu_chpl.chpl) with the same Pool contract: step 1 on the CPU, step 2 on D tasks, step 3 on the CPU.
// part < 0: the whole search.  part >= 0: only task `part` of the D-way static split, on `device` (one rank of a
// process-per-GPU launch): the step-1 tree is credited to part 0 and every part drains its own leftovers, so the
// per-part counts add up to the whole search's.  `on` != nullptr: D = 1 on device pools of a handle the caller created
// (set-up outside the search's timers, as the Chapel drivers' `on device var` declarations are).
// `ck` (D tasks on device or host pools, part < 0): a resumed search skips step 1 and continues step 2 from the
// checkpoint; a search that stops writes the checkpoint and returns TSB_ESTOPPED with the counts so far.
template <class S>
int three_step_search(const S& s, int m, int M, int D, int part, int device, typename S::Handle* on,
                      tsb_search_stats* out, SearchCkpt* ck = nullptr) {
  using Node = typename S::Node;
  const tsb::ckpt::State* from = ck ? ck->resume : nullptr;
  if (from && s.steal && D > 1)  // (tasks that steal leave step 2 together: none can have finished alone)
    for (const auto& t : from->tasks)
      if (t.finished) return TSB_EINVAL;
  if (!on)
    if (int rc = tsb_init_devices(part < 0 ? D : device + 1); rc != TSB_OK) return rc;  // contexts exist before the timers start
  int64_t best = s.initial_best;
  Pool<Node> pool;
  if (!from) pool.pushBack(s.root());
  uint64_t tree = 0, sol = 0;
  Node parent;
  double t0 = now_s();
  while (pool.size < static_cast<size_t>(D) * m * s.pools) {  // step 1 (nqueens_multigpu_chpl.chpl:173-179)
    if (!pool.popFront(parent)) break;
    s.decompose(parent, tree, sol, best, pool);
  }
  double t1 = now_s();
  out->t_step1 = t1 - t0;
  std::vector<GpuTaskResult> res(D);
  std::vector<TaskCkpt> tck(ck ? D : 0);
  for (TaskCkpt& t : tck) t.stop = &ck->stop;
  if (from) {  // step 1 and the tasks' counters as the checkpoint has them
    tree = from->tree1;
    sol = from->sol1;
    best = from->best1;
    out->t_step1 = from->t_step1;
    for (int gid = 0; gid < D; gid++) {
      const tsb::ckpt::TaskState& t = from->tasks[gid];
      GpuTaskResult& r = res[gid];
      r.tree = t.tree, r.sol = t.sol, r.offloads = t.offloads, r.parents = t.parents, r.launches = t.launches;
      if (!t.finished) tck[gid].resume = &t.pools;
    }
  }
  // step 2: on device pools, every task's pool moves to its device and stays there; tasks that run dry steal from
  // the fullest device pool peer-to-peer
  for (auto& r : res) r.best = best;  // per-task best_l = best (pfsp_multigpu_chpl.chpl:384)
  if (from)
    for (int gid = 0; gid < D; gid++) res[gid].best = from->tasks[gid].best;
  // a task that had left step 2 when the checkpoint was written does not run again: its host pool holds its leftovers
  const auto finished = [&](int gid) { return from && from->tasks[gid].finished; };
  const auto task = [&](int dev, Pool<Node>& own, GpuTaskResult& r, StealBoard* sb, int me) {
    if (finished(me)) {
      push_records(from->tasks[me].left, own);
    } else if (s.devpool) {
      s.device_task(dev, m, M, own, r, sb, me, ck ? &tck[me] : nullptr);
    } else {
      s.host_task(dev, m, M, own, r, ck ? &tck[me] : nullptr);
    }
  };
  // a task's leftovers back to the global pool (:315-320); several pools per task already handed theirs back to the
  // task's pool one by one, as the reference's tasks do, so that order stays
  const auto hand_back = [&](Pool<Node>& from) {
    if (s.pools > 1)
      for (size_t i = 0; i < from.size; i++) pool.pushBack(from.el[from.front + i]);
    else
      while (from.popBack(parent)) pool.pushBack(parent);
  };
  // task g drives GPU g; with fewer than D GPUs present the tasks wrap around (g % ndev): the
  // per-task pools stay independent, so counts are unchanged — used to test D > 1 on one GPU
  const int ndev = std::max(1, tsb_device_count());
  std::vector<Pool<Node>> multi;
  bool stopped = false;  // (a resumable search: some task stopped for the checkpoint)
  if (on) {
    devpool_on(s, on, m, M, pool, res[0], nullptr, 0, nullptr);
  } else if (part >= 0) {
    if (part != 0) tree = sol = 0;  // step 1 is credited to part 0
    static_split(pool, D, multi);
    task(device, multi[part], res[part], nullptr, 0);
    hand_back(multi[part]);
  } else if (D == 1) {
    task(0, pool, res[0], nullptr, 0);
    stopped = ck && tck[0].stopped;
  } else {
    static_split(pool, D, multi);
    StealBoard board(D);
    StealBoard* sb = s.steal ? &board : nullptr;
    std::vector<std::thread> th;
    for (int gid = 0; gid < D; gid++)
      th.emplace_back([&, gid] {
        if (finished(gid)) return task(gid, multi[gid], res[gid], nullptr, gid);
        bind_task(gid % ndev);
        task(gid % ndev, multi[gid], res[gid], sb, gid);
      });
    for (auto& x : th) x.join();
    for (const TaskCkpt& t : tck) stopped = stopped || t.stopped;
    for (int gid = 0; gid < D && !stopped; gid++) hand_back(multi[gid]);
    out->steals = (from ? from->steals : 0) + board.steals;
  }
  const uint64_t tree1 = tree, sol1 = sol;
  const int64_t best1 = best;
  for (int gid = 0; gid < D; gid++) {
    if (res[gid].rc != TSB_OK) return res[gid].rc;
    tree += res[gid].tree;
    sol += res[gid].sol;
    best = std::min(best, res[gid].best);  // min reduce (pfsp_multigpu_chpl.chpl:520)
    out->offloads += res[gid].offloads;
    out->offloaded_parents += res[gid].parents;
    out->kernel_launches += res[gid].launches;
    out->per_gpu_tree[gid] = res[gid].tree;
  }
  double t2 = now_s();
  out->t_step2 = (from ? from->t_step2 : 0) + (t2 - t1);
  if (stopped) {  // the checkpoint: step 1, every task's counters, and its pools or (finished) its leftovers
    tsb::ckpt::State st;
    st.p = ck->params;
    st.tree1 = tree1, st.sol1 = sol1, st.best1 = best1;
    st.t_step1 = out->t_step1, st.t_step2 = out->t_step2, st.steals = out->steals;
    st.tasks.resize(D);
    for (int gid = 0; gid < D; gid++) {
      const GpuTaskResult& r = res[gid];
      tsb::ckpt::TaskState& t = st.tasks[gid];
      t.tree = r.tree, t.sol = r.sol, t.offloads = r.offloads, t.parents = r.parents, t.launches = r.launches;
      t.best = r.best;
      t.finished = !tck[gid].stopped;
      if (t.finished) {
        t.left = pool_records(D == 1 ? pool : multi[gid]);
      } else {
        t.pools = std::move(tck[gid].pools);
      }
    }
    const double tw = now_s();
    if (int rc = tsb::ckpt::save(ck->path, st); rc != TSB_OK) return rc;
    if (std::getenv("TSB200_TRACE")) {
      size_t nodes = 0;
      for (const auto& t : st.tasks) {
        nodes += t.left.size();
        for (const auto& x : t.pools) nodes += x.nodes.size();
      }
      std::fprintf(stderr, "[tsb200] checkpoint: %zu nodes written in %.1f ms\n", nodes / sizeof(Node),
                   (now_s() - tw) * 1e3);
    }
    out->explored_tree = tree;
    out->explored_sol = sol;
    out->best = best;
    return TSB_ESTOPPED;
  }
  while (pool.popBack(parent)) s.decompose(parent, tree, sol, best, pool);  // step 3
  out->t_step3 = now_s() - t2;
  out->explored_tree = tree;
  out->explored_sol = sol;
  out->best = best;
  return TSB_OK;
}

template <class Node>
int nq_search(int N, int g, int m, int M, int D, bool devpool, int part, int device, tsb_nq* on,
              tsb_search_stats* out, SearchCkpt* ck = nullptr) {
  constexpr bool wide = std::is_same_v<Node, tsb_nq_node24>;
  if (!out || N < 1 || N > (wide ? TSB_MAX_QUEENS_WIDE : TSB_MAX_QUEENS) || g < 1 || m < 1 || M < 1 || D < 1 || D > 8 ||
      part >= D)
    return TSB_EINVAL;
  std::memset(out, 0, sizeof(*out));
  return three_step_search(NqSearch<Node>(N, g, M, devpool), m, M, D, part, device, on, out, ck);
}

inline int pfsp_tables_for(tsb_pfsp_tables* t, int inst) { return tsb_pfsp_tables_build(t, inst); }
inline int pfsp_tables_for(tsb_pfsp_tables50* t, int inst) {
  // (the 50-job instances only: tsb_pfsp_tables50_build also takes the smaller ones)
  if (inst < 31 || inst > 60) return TSB_EUNSUPPORTED;
  return tsb_pfsp_tables50_build(t, inst, TSB_LB2_FULL);
}

// pools > 1 (device pools only): every task's share split once more into `pools` device pools (devpool_on).
// Node: tsb_pfsp_node (a MAX_JOBS = 20 build) or tsb_pfsp_node50 (MAX_JOBS = 50, ta031..ta060).
template <class Node = tsb_pfsp_node>
int pfsp_search(int inst, int lb_kind, int ub, int m, int M, int D, bool devpool, int part, int device, tsb_pfsp* on,
                tsb_search_stats* out, int pools = 1, SearchCkpt* ck = nullptr) {
  using Tables = std::conditional_t<std::is_same_v<Node, tsb_pfsp_node50>, tsb_pfsp_tables50, tsb_pfsp_tables>;
  if (!out || lb_kind < 0 || lb_kind > 2 || (ub != 0 && ub != 1) || m < 1 || M < 1 || D < 1 || D > 8 || part >= D ||
      pools < 1 || pools > 4)
    return TSB_EINVAL;
  std::memset(out, 0, sizeof(*out));
  std::vector<Tables> tv(1);
  if (int rc = pfsp_tables_for(&tv[0], inst); rc != TSB_OK) return rc;
  return three_step_search(PfspSearch<Node, Tables>(tv[0], inst, lb_kind, ub, devpool, pools), m, M, D, part, device,
                           on, out, ck);
}

// the resumable searches: resume from `path` if a checkpoint is there (refused before any device call if it is damaged
// or was written for other parameters), run `run` under a stop condition, remove the checkpoint when the search ends
template <class Run>
int ckpt_search(const char* path, double seconds, const tsb::ckpt::Params& p, Run&& run) {
  if (!path || !*path || std::isnan(seconds)) return TSB_EINVAL;
  tsb::ckpt::State st;
  const double t0 = now_s();
  const int got = tsb::ckpt::load(path, p, &st);
  if (got < 0) return got;
  if (got && std::getenv("TSB200_TRACE")) std::fprintf(stderr, "[tsb200] checkpoint: read in %.1f ms\n", (now_s() - t0) * 1e3);
  SearchCkpt ck{path, p, got ? &st : nullptr, {}};
  ck.stop.deadline = seconds < 0 ? HUGE_VAL : now_s() + seconds;
  const int rc = run(&ck);
  if (rc == TSB_OK) std::remove(path);
  if (rc == TSB_ESTOPPED) g_stop_request.store(0);
  return rc;
}

template <class Node>
int nq_warmup(int N, int min_size, void* nodes, int64_t capacity, int64_t* n, uint64_t* tree, uint64_t* sol) {
  if (min_size < 1 || !n || !tree || !sol || (capacity && !nodes)) return TSB_EINVAL;
  Pool<Node> pool;
  Node root{}, parent;
  for (int i = 0; i < N; i++) root.board[i] = static_cast<uint8_t>(i);
  pool.pushBack(root);
  *tree = *sol = 0;
  while (pool.size < static_cast<size_t>(min_size)) {
    if (!pool.popFront(parent)) break;
    nq_decompose(N, parent, *tree, *sol, pool);
  }
  *n = static_cast<int64_t>(pool.size);
  if (*n > capacity) return TSB_ENOMEM;
  if (pool.size) std::memcpy(nodes, &pool.el[pool.front], pool.size * sizeof(Node));
  return TSB_OK;
}
// the search's node type for N (whole searches: the wide records only where the narrow ones cannot hold the board)
template <class F>
int with_nq_node(bool wide, F&& f) {
  return wide ? f(tsb_nq_node24{}) : f(tsb_nq_node{});
}

// tsb_nq_search[_device]_ckpt: max_queens = 20 runs N <= 20 on 21-byte nodes and N > 20 on 25-byte nodes, 24 every N
// on 25-byte nodes.  (N-Queens has no pools argument: how many device pools a task runs is checked against the
// checkpoint per task; c = 1 marks the host-pool search, search_ckpt.h)
int nq_search_ckpt(bool devpool, int max_queens, int N, int g, int m, int M, int D, const char* path, double seconds,
                   tsb_search_stats* out) {
  if (max_queens != TSB_MAX_QUEENS && max_queens != TSB_MAX_QUEENS_WIDE) return TSB_EINVAL;
  return with_nq_node(max_queens == TSB_MAX_QUEENS_WIDE || N > TSB_MAX_QUEENS, [&](auto node) {
    using Node = decltype(node);
    const tsb::ckpt::Params p{tsb::ckpt::kNQueens, sizeof(Node), N, g, devpool ? 0 : 1, m, M, D, 0};
    return ckpt_search(path, seconds, p, [&](SearchCkpt* ck) {
      return nq_search<Node>(N, g, m, M, D, devpool, -1, 0, nullptr, out, ck);
    });
  });
}
// tsb_pfsp_search[_device]_ckpt[_wide]: the host-pool search has one pool per task and writes pools = 0
template <class Node>
int pfsp_search_ckpt(bool devpool, int inst, int lb_kind, int ub, int m, int M, int D, int pools, const char* path,
                     double seconds, tsb_search_stats* out) {
  const tsb::ckpt::Params p{tsb::ckpt::kPfsp, sizeof(Node), inst, lb_kind, ub, m, M, D, devpool ? pools : 0};
  return ckpt_search(path, seconds, p, [&](SearchCkpt* ck) {
    return pfsp_search<Node>(inst, lb_kind, ub, m, M, D, devpool, -1, 0, nullptr, out, pools, ck);
  });
}
}  // namespace

// ====================================================================== exported
extern "C" {

int tsb_taillard_nb_jobs(int id) {
  return id > 110 ? 500 : id > 90 ? 200 : id > 60 ? 100 : id > 30 ? 50 : 20;
}
int tsb_taillard_nb_machines(int id) {
  static const int m[12] = {5, 10, 20, 5, 10, 20, 5, 10, 20, 10, 20, 20};  // per group of ten instances
  if (id < 1 || id > 120) return -1;
  return m[(id - 1) / 10];
}
int64_t tsb_taillard_best_ub(int id) { return (id < 1 || id > 120) ? -1 : kBestUb[id - 1]; }

int tsb_pfsp_tables_build(tsb_pfsp_tables* t, int inst) { return tsb_pfsp_tables_build_variant(t, inst, TSB_LB2_FULL); }
int tsb_pfsp_tables_build_variant(tsb_pfsp_tables* t, int inst, int variant) {
  return build_tables<tsb_pfsp_tables, TSB_MAX_JOBS>(t, inst, variant);
}
int tsb_pfsp_tables50_build(tsb_pfsp_tables50* t, int inst, int variant) {
  return build_tables<tsb_pfsp_tables50, TSB_MAX_JOBS_WIDE>(t, inst, variant);
}
int tsb_pfsp_create50_from_tables(tsb_pfsp** h, int device, int M_max, const tsb_pfsp_tables50* t) {
  if (!t) return TSB_EINVAL;
  return tsb_pfsp_create_wide(h, device, TSB_MAX_JOBS_WIDE, t->jobs, t->machines, M_max, t->p_times, t->min_heads,
                              t->min_tails, t->pairs, t->johnson, t->lags, t->mp0, t->mp1, t->mp_order);
}

int tsb_pfsp_create_from_tables(tsb_pfsp** h, int device, int M_max, const tsb_pfsp_tables* t) {
  if (!t) return TSB_EINVAL;
  return tsb_pfsp_create(h, device, t->jobs, t->machines, M_max, t->p_times, t->min_heads, t->min_tails,
                         t->pairs, t->johnson, t->lags, t->mp0, t->mp1, t->mp_order);
}

void tsb_release_cached_handles(void) { nq_handle_cache().clear(); }

// step 1 of the drivers alone (nqueens_gpu_chpl.chpl:169-175): breadth-first from the root until the pool holds
// min_size nodes; the pool, in order, and what was explored on the way
int tsb_nq_warmup(int N, int min_size, void* nodes, int64_t capacity, int64_t* n, uint64_t* tree, uint64_t* sol) {
  if (N < 1 || N > TSB_MAX_QUEENS_WIDE) return TSB_EINVAL;
  return with_nq_node(N > TSB_MAX_QUEENS, [&](auto node) {
    return nq_warmup<decltype(node)>(N, min_size, nodes, capacity, n, tree, sol);
  });
}

int tsb_nq_search(int N, int g, int m, int M, int D, tsb_search_stats* out) {
  return with_nq_node(N > TSB_MAX_QUEENS, [&](auto node) {
    return nq_search<decltype(node)>(N, g, m, M, D, false, -1, 0, nullptr, out);
  });
}
int tsb_nq_search_wide(int max_queens, int N, int g, int m, int M, int D, tsb_search_stats* out) {
  if (max_queens != TSB_MAX_QUEENS_WIDE) return TSB_EINVAL;
  return nq_search<tsb_nq_node24>(N, g, m, M, D, false, -1, 0, nullptr, out);
}
int tsb_nq_search_device(int N, int g, int m, int M, int D, tsb_search_stats* out) {
  return with_nq_node(N > TSB_MAX_QUEENS, [&](auto node) {
    return nq_search<decltype(node)>(N, g, m, M, D, true, -1, 0, nullptr, out);
  });
}
int tsb_nq_search_device_wide(int max_queens, int N, int g, int m, int M, int D, tsb_search_stats* out) {
  if (max_queens != TSB_MAX_QUEENS_WIDE) return TSB_EINVAL;
  return nq_search<tsb_nq_node24>(N, g, m, M, D, true, -1, 0, nullptr, out);
}
int tsb_nq_search_device_part(int N, int g, int m, int M, int D, int part, int device, tsb_search_stats* out) {
  if (part < 0) return TSB_EINVAL;
  return with_nq_node(N > TSB_MAX_QUEENS, [&](auto node) {
    return nq_search<decltype(node)>(N, g, m, M, D, true, part, device, nullptr, out);
  });
}
int tsb_nq_search_on(tsb_nq* h, int N, int m, int M, tsb_search_stats* out) {
  if (!h) return TSB_EINVAL;
  return with_nq_node(tsb_nq_max_queens(h) == TSB_MAX_QUEENS_WIDE, [&](auto node) {
    return nq_search<decltype(node)>(N, 1, m, M, 1, true, -1, 0, h, out);
  });
}
int tsb_pfsp_search(int inst, int lb_kind, int ub, int m, int M, int D, tsb_search_stats* out) {
  return pfsp_search(inst, lb_kind, ub, m, M, D, false, -1, 0, nullptr, out);
}
int tsb_pfsp_search_device(int inst, int lb_kind, int ub, int m, int M, int D, tsb_search_stats* out) {
  return pfsp_search(inst, lb_kind, ub, m, M, D, true, -1, 0, nullptr, out);
}
int tsb_pfsp_search_device_part(int inst, int lb_kind, int ub, int m, int M, int D, int part, int device,
                                tsb_search_stats* out) {
  if (part < 0) return TSB_EINVAL;
  return pfsp_search(inst, lb_kind, ub, m, M, D, true, part, device, nullptr, out);
}
int tsb_pfsp_search_on(tsb_pfsp* h, int inst, int lb_kind, int ub, int m, int M, tsb_search_stats* out) {
  if (!h) return TSB_EINVAL;
  return pfsp_search(inst, lb_kind, ub, m, M, 1, true, -1, 0, h, out);
}
int tsb_pfsp_search_device_pools(int inst, int lb_kind, int ub, int m, int M, int D, int pools, tsb_search_stats* out) {
  return pfsp_search(inst, lb_kind, ub, m, M, D, true, -1, 0, nullptr, out, pools);
}
int tsb_pfsp_search_device_pools_part(int inst, int lb_kind, int ub, int m, int M, int D, int pools, int part,
                                      int device, tsb_search_stats* out) {
  if (part < 0) return TSB_EINVAL;
  return pfsp_search(inst, lb_kind, ub, m, M, D, true, part, device, nullptr, out, pools);
}
int tsb_pfsp_search_on_pools(tsb_pfsp* h, int inst, int lb_kind, int ub, int m, int M, int pools,
                             tsb_search_stats* out) {
  if (!h) return TSB_EINVAL;
  return pfsp_search(inst, lb_kind, ub, m, M, 1, true, -1, 0, h, out, pools);
}

int tsb_nq_search_device_ckpt(int max_queens, int N, int g, int m, int M, int D, const char* path, double seconds,
                              tsb_search_stats* out) {
  return nq_search_ckpt(true, max_queens, N, g, m, M, D, path, seconds, out);
}
int tsb_nq_search_ckpt(int max_queens, int N, int g, int m, int M, int D, const char* path, double seconds,
                       tsb_search_stats* out) {
  return nq_search_ckpt(false, max_queens, N, g, m, M, D, path, seconds, out);
}
int tsb_pfsp_search_device_ckpt(int inst, int lb_kind, int ub, int m, int M, int D, int pools, const char* path,
                                double seconds, tsb_search_stats* out) {
  return pfsp_search_ckpt<tsb_pfsp_node>(true, inst, lb_kind, ub, m, M, D, pools, path, seconds, out);
}
int tsb_pfsp_search_ckpt(int inst, int lb_kind, int ub, int m, int M, int D, const char* path, double seconds,
                         tsb_search_stats* out) {
  return pfsp_search_ckpt<tsb_pfsp_node>(false, inst, lb_kind, ub, m, M, D, 1, path, seconds, out);
}
int tsb_pfsp_search_wide(int max_jobs, int inst, int lb_kind, int ub, int m, int M, int D, tsb_search_stats* out) {
  if (max_jobs != TSB_MAX_JOBS_WIDE) return TSB_EINVAL;
  return pfsp_search<tsb_pfsp_node50>(inst, lb_kind, ub, m, M, D, false, -1, 0, nullptr, out);
}
int tsb_pfsp_search_device_wide(int max_jobs, int inst, int lb_kind, int ub, int m, int M, int D, int pools,
                                tsb_search_stats* out) {
  if (max_jobs != TSB_MAX_JOBS_WIDE) return TSB_EINVAL;
  return pfsp_search<tsb_pfsp_node50>(inst, lb_kind, ub, m, M, D, true, -1, 0, nullptr, out, pools);
}
int tsb_pfsp_search_device_ckpt_wide(int max_jobs, int inst, int lb_kind, int ub, int m, int M, int D, int pools,
                                     const char* path, double seconds, tsb_search_stats* out) {
  if (max_jobs != TSB_MAX_JOBS_WIDE) return TSB_EINVAL;
  return pfsp_search_ckpt<tsb_pfsp_node50>(true, inst, lb_kind, ub, m, M, D, pools, path, seconds, out);
}
int tsb_pfsp_search_ckpt_wide(int max_jobs, int inst, int lb_kind, int ub, int m, int M, int D, const char* path,
                              double seconds, tsb_search_stats* out) {
  if (max_jobs != TSB_MAX_JOBS_WIDE) return TSB_EINVAL;
  return pfsp_search_ckpt<tsb_pfsp_node50>(false, inst, lb_kind, ub, m, M, D, 1, path, seconds, out);
}
void tsb_search_request_stop(void) { g_stop_request.store(1); }

}  // extern "C"

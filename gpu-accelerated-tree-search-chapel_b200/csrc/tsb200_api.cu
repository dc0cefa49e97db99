// tsb200_api.cu — C ABI of libtsb200.so (include/tsb200.h): handles, transfers, kernel launches.
#include <cuda_runtime.h>

#include <sched.h>

#include <algorithm>
#include <cctype>
#include <atomic>
#include <chrono>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <type_traits>
#include <vector>

#include "xfer_route.h"
#include "nq_expand.cuh"
#include "nq_rounds_ll.cuh"
#include "pfsp_expand.cuh"
#include "pfsp_rounds.cuh"
#include "nq_kernel.cuh"
#include "pfsp_kernels.cuh"
#include "pfsp_wide.cuh"
#include "pfsp_wide_expand.cuh"
#include "pfsp_wide_rounds.cuh"
#include "pfsp_search_pool.h"
#include "tsb200.h"

// Internals shared by both handle types (the handles themselves are the header's types, defined after this block)
namespace {

thread_local std::string g_last_cuda_error;

#define TSB_CUDA(call)                                                                         \
  do {                                                                                         \
    cudaError_t e__ = (call);                                                                  \
    if (e__ != cudaSuccess) {                                                                  \
      g_last_cuda_error = std::string(#call) + ": " + cudaGetErrorString(e__);                 \
      (void)cudaGetLastError();                                                                \
      return e__ == cudaErrorMemoryAllocation ? TSB_ENOMEM : TSB_ECUDA;                        \
    }                                                                                          \
  } while (0)

// (env TSB200_POOL_CAP overrides the initial arena capacity, so that tests can force compaction and growth)
long long env_pool_cap() {
  const char* v = std::getenv("TSB200_POOL_CAP");
  return v ? std::atoll(v) : 0;
}
int env_xfer() {
  const char* s = std::getenv("TSB200_XFER");
  if (!s) return TSB_XFER_AUTO;
  if (!std::strcmp(s, "memcpy")) return TSB_XFER_MEMCPY;
  if (!std::strcmp(s, "zerocopy")) return TSB_XFER_ZEROCOPY;
  return TSB_XFER_AUTO;
}
bool env_no_register() {
  const char* s = std::getenv("TSB200_NO_REGISTER");
  return s && *s && *s != '0';
}
bool env_no_rounds() {
  const char* v = std::getenv("TSB200_NO_ROUNDS");
  return v && *v && *v != '0';
}

// Host ranges the CALLER asked to page-lock + map (tsb_*_register_host): cudaMemcpyAsync is truly asynchronous
// on them and the zero-copy kernels can address them.  Registration is explicit and the caller owns the
// lifetime: a range must stay allocated until it is unregistered or the handle is destroyed (a registration
// keyed on an address alone goes stale when the array is freed and another one lands on the same addresses).
// Arrays that were never registered go through the handle's own pinned staging buffers.
struct HostRange {
  uintptr_t base;
  size_t len;
};
struct HostRegistry {
  std::vector<HostRange> ranges;
  bool disabled = env_no_register();
  bool contains(const void* p, size_t bytes) const {
    if (!p || !bytes) return false;
    const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = a + bytes;
    for (const auto& r : ranges)
      if (a >= r.base && b <= r.base + r.len) return true;
    return false;
  }
  // TSB_OK, or TSB_EINVAL for a range that partly overlaps a registered one, or TSB_ECUDA
  int add(void* p, size_t bytes) {
    if (!p || !bytes) return TSB_EINVAL;
    if (disabled || contains(p, bytes)) return TSB_OK;
    const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = a + bytes;
    for (const auto& r : ranges)
      if (r.base < b && a < r.base + r.len) return TSB_EINVAL;
    TSB_CUDA(cudaHostRegister(p, bytes, cudaHostRegisterPortable | cudaHostRegisterMapped));
    ranges.push_back({a, bytes});
    return TSB_OK;
  }
  int remove(void* p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    for (size_t i = 0; i < ranges.size(); i++)
      if (ranges[i].base == a) {
        cudaHostUnregister(p);
        ranges.erase(ranges.begin() + i);
        return TSB_OK;
      }
    return disabled ? TSB_OK : TSB_EINVAL;
  }
  void release() {
    for (auto& r : ranges) cudaHostUnregister(reinterpret_cast<void*>(r.base));
    ranges.clear();
  }
};

struct DeviceInfo {
  int sms = 0;
  bool can_use_host_ptr = false;
  bool coop = false;  // cooperative launches (the persistent multi-round kernel)
};
int query_device(int device, DeviceInfo& di) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    (void)cudaGetLastError();
    return TSB_ENODEV;
  }
  if (device < 0 || device >= n) return TSB_ENODEV;
  TSB_CUDA(cudaSetDevice(device));
  TSB_CUDA(cudaDeviceGetAttribute(&di.sms, cudaDevAttrMultiProcessorCount, device));
  int v = 0;
  TSB_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrCanUseHostPointerForRegisteredMem, device));
  di.can_use_host_ptr = v != 0;
  TSB_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrCooperativeLaunch, device));
  di.coop = v != 0;
  return TSB_OK;
}

struct PoolExtent {
  long long b, e;  // arena positions [b, e)
};

// Device-resident pool: a stack of extents inside one arena of `rec`-byte nodes.  A round reads the newest
// nodes in place (possibly spanning several extents) and appends the children above the top, so nothing is
// copied; the holes left behind are reclaimed by compacting into the second arena when the top reaches the end.
struct DevicePool {
  uint8_t* arena[2] = {nullptr, nullptr};
  long long cap = 0;  // nodes per arena
  int cur = 0;
  std::vector<PoolExtent> ext;
  long long size = 0;
  // the node format (set_format)
  size_t rec = 0, slack = 0;
  long long align = 1;        // extents start at a multiple of `align` records
  int fanout = 0;             // most children one node can have
  long long default_cap = 0;  // nodes the arena starts with

  // `node_bytes`-byte nodes read in tiles of `tile` records (full-tile loads may run past the top)
  void set_format(size_t node_bytes, int tile, long long node_align, int max_children, long long start_cap) {
    rec = node_bytes;
    slack = static_cast<size_t>(tile) * node_bytes;
    align = node_align;
    fanout = max_children;
    default_cap = start_cap;
  }
  // (read when the arena is first allocated: the search drivers keep handles between searches)
  long long min_cap() const {
    if (const long long c = env_pool_cap(); c > 0) return c;
    return default_cap;
  }
  long long top() const { return ext.empty() ? 0 : ext.back().e; }
  // where the next extent may start
  long long aligned_top() const { return (top() + align - 1) / align * align; }
  size_t bytes(long long nodes) const { return static_cast<size_t>(nodes) * rec + slack + 64; }
  int ensure_arena(int which) {
    if (!arena[which]) TSB_CUDA(cudaMalloc(&arena[which], bytes(cap)));
    return TSB_OK;
  }
  // all extents -> [0, size) of the other arena (or of fresh, larger arenas when `new_cap` > cap)
  int compact(cudaStream_t s, long long new_cap) {
    uint8_t* dst = nullptr;
    const bool grow = new_cap > cap;
    if (grow) {
      TSB_CUDA(cudaMalloc(&dst, bytes(new_cap)));
    } else {
      int rc = ensure_arena(cur ^ 1);
      if (rc != TSB_OK) return rc;
      dst = arena[cur ^ 1];
    }
    long long at = 0;
    for (const PoolExtent& x : ext) {
      TSB_CUDA(cudaMemcpyAsync(dst + at * rec, arena[cur] + x.b * rec, static_cast<size_t>(x.e - x.b) * rec,
                               cudaMemcpyDeviceToDevice, s));
      at += x.e - x.b;
    }
    TSB_CUDA(cudaStreamSynchronize(s));
    if (grow) {
      for (int i = 0; i < 2; i++) {
        if (arena[i]) cudaFree(arena[i]);
        arena[i] = nullptr;
      }
      arena[0] = dst;
      cur = 0;
      cap = new_cap;
    } else {
      cur ^= 1;
    }
    ext.clear();
    if (at) ext.push_back({0, at});
    return TSB_OK;
  }
  // room for `extra` nodes above the top
  int reserve(cudaStream_t s, long long extra) {
    if (cap == 0) {
      cap = std::max<long long>(min_cap(), extra + 1024);
      int rc = ensure_arena(cur);
      if (rc != TSB_OK) return rc;
    }
    if (top() + extra <= cap) return TSB_OK;
    const long long need = size + extra;
    return compact(s, need > cap ? std::max<long long>(2 * cap, need + need / 2) : cap);
  }
  // the pool as ONE contiguous stack [0, size) in an arena of at least `need` nodes (the persistent kernels' layout)
  int make_stack(cudaStream_t s, long long need) {
    if (need > cap) return compact(s, std::max<long long>(2 * cap, need + need / 2));
    if (ext.size() != 1 || ext[0].b != 0) return compact(s, cap);
    return TSB_OK;
  }
  // a persistent launch left the pool as the stack [0, n)
  void set_stack(long long n) {
    size = n;
    ext.clear();
    if (n) ext.push_back({0, n});
  }
  // the newest n nodes, as pieces in logical order
  void top_pieces(long long n, std::vector<PoolExtent>* pieces) const {
    pieces->clear();
    long long left = n;
    for (size_t i = ext.size(); i-- > 0 && left > 0;) {
      const long long t = std::min(left, ext[i].e - ext[i].b);
      pieces->insert(pieces->begin(), PoolExtent{ext[i].e - t, ext[i].e});
      left -= t;
    }
  }
  // drop the newest n nodes
  void pop(long long n) {
    long long left = n;
    while (left > 0 && !ext.empty()) {
      PoolExtent& x = ext.back();
      const long long t = std::min(left, x.e - x.b);
      x.e -= t;
      left -= t;
      if (x.e == x.b) ext.pop_back();
    }
    size -= n;
  }
  // n nodes written at [at, at + n) become the newest extent
  void push_extent(long long at, long long n) {
    if (!n) return;
    ext.push_back({at, at + n});
    size += n;
  }
  void release() {
    for (int i = 0; i < 2; i++) {
      if (arena[i]) cudaFree(arena[i]);
      arena[i] = nullptr;
    }
    ext.clear();
    size = 0;
    cap = 0;
  }
};

// state of the fused expand kernels of one handle (expand_common.cuh)
struct ExpandCtx {
  uint32_t* d_cmask = nullptr;  // side array of the round, `side_bytes` per tile: PFSP: one child mask per parent;
                                // N-Queens: the tile's items (one uint16 per child)
  int* d_tile = nullptr;        // per-tile child counts
  long long tile_cap = 0;       // tiles the two arrays above hold
  long long side_bytes = 0;
  tsb::ExpandState* d_st = nullptr;
  tsb::ExpandResult* h_res = nullptr;  // pinned + mapped: written by the scan kernel of a round
  tsb::ExpandResult* d_res = nullptr;  // device alias of h_res
  unsigned epoch = 0;
  // (clears are ordered on the stream the kernels run on: the handle's streams do not synchronise with the
  // legacy default stream)
  int reserve(long long tiles, long long side_bytes_per_tile, cudaStream_t s, int best_init = 0x7FFFFFFF) {
    if (!d_st) {
      TSB_CUDA(cudaMalloc(&d_st, sizeof(tsb::ExpandState)));
      const tsb::ExpandState init{0ull, best_init, 0};
      TSB_CUDA(cudaMemcpyAsync(d_st, &init, sizeof(init), cudaMemcpyHostToDevice, s));
      TSB_CUDA(cudaStreamSynchronize(s));  // `init` lives on this stack frame
    }
    if (!h_res) {
      TSB_CUDA(cudaHostAlloc(&h_res, sizeof(tsb::ExpandResult), cudaHostAllocPortable | cudaHostAllocMapped));
      // (epochs start at 1: recycled pinned memory may hold another handle's old record, epoch included — the early
      // wait below would take it for this handle's first round)
      std::memset(h_res, 0, sizeof(tsb::ExpandResult));
      TSB_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&d_res), h_res, 0));
    }
    if (tiles > tile_cap || side_bytes_per_tile > side_bytes) {
      side_bytes_per_tile = std::max(side_bytes_per_tile, side_bytes);
      if (d_cmask) cudaFree(d_cmask);
      if (d_tile) cudaFree(d_tile);
      d_cmask = nullptr;
      d_tile = nullptr;
      tile_cap = 0;
      const long long cap = std::max<long long>(tiles + tiles / 4 + 16, 1024);
      TSB_CUDA(cudaMalloc(&d_cmask, static_cast<size_t>(cap) * side_bytes_per_tile + 64));
      TSB_CUDA(cudaMalloc(&d_tile, static_cast<size_t>(cap) * sizeof(int)));
      tile_cap = cap;
      side_bytes = side_bytes_per_tile;
    }
    return TSB_OK;
  }
  // Wait for the round's result record.  `early`: return as soon as the build kernel's first CTA has published
  // the counts (it does so in its prologue) — the children are still being written, which is fine for a caller
  // whose next use of them is ordered on the same stream (the pool); the host then prepares and launches the next
  // round while this one finishes, which hides the launch + synchronisation latency of small rounds.
  int wait_result(unsigned want_epoch, cudaStream_t s, bool early) {
    if (early) {
      const volatile unsigned long long* ep = &h_res->epoch;
      for (unsigned spin = 0;; spin++) {
        if (*ep == want_epoch) return TSB_OK;
        if ((spin & 1023u) == 1023u) {  // a faulted kernel never publishes: ask the stream now and then
          const cudaError_t q = cudaStreamQuery(s);
          if (q == cudaSuccess) return *ep == want_epoch ? TSB_OK : TSB_ECUDA;
          if (q != cudaErrorNotReady) {
            g_last_cuda_error = std::string("expand kernels: ") + cudaGetErrorString(q);
            (void)cudaGetLastError();
            return TSB_ECUDA;
          }
        }
      }
    }
    TSB_CUDA(cudaStreamSynchronize(s));
    return h_res->epoch == want_epoch ? TSB_OK : TSB_ECUDA;
  }
  void release() {
    if (d_cmask) cudaFree(d_cmask);
    if (d_tile) cudaFree(d_tile);
    if (d_st) cudaFree(d_st);
    if (h_res) cudaFreeHost(h_res);
    d_cmask = nullptr;
    d_tile = nullptr;
    d_st = nullptr;
    h_res = d_res = nullptr;
  }
};

// state of the persistent multi-round kernel of one handle (nq_rounds_ll.cuh, pfsp_rounds.cuh)
struct RoundsCtx {
  tsb::RoundsState* h_state = nullptr;  // pinned + mapped: written by the kernel when it leaves
  tsb::RoundsState* d_state = nullptr;  // device alias of h_state
  void* d_sync = nullptr;               // the kernel's exchange flags: tsb::LlSync or tsb::PfRoundsSync
  unsigned epoch = 0;                   // epoch the last launch left the flags at
  template <class Sync>
  int ensure(cudaStream_t s) {
    if (!h_state) {
      TSB_CUDA(cudaHostAlloc(&h_state, sizeof(tsb::RoundsState), cudaHostAllocPortable | cudaHostAllocMapped));
      std::memset(h_state, 0, sizeof(tsb::RoundsState));
      TSB_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&d_state), h_state, 0));
    }
    if (!d_sync) {
      TSB_CUDA(cudaMalloc(&d_sync, sizeof(Sync)));
      TSB_CUDA(cudaMemsetAsync(d_sync, 0, sizeof(Sync), s));
    }
    return TSB_OK;
  }
  template <class Sync>
  Sync* sync() const {
    return static_cast<Sync*>(d_sync);
  }
  void release() {
    if (h_state) cudaFreeHost(h_state);
    if (d_sync) cudaFree(d_sync);
    h_state = d_state = nullptr;
    d_sync = nullptr;
  }
};

// common part of both handle types
struct Base {
  int device = 0, M_max = 0, xfer = TSB_XFER_AUTO;
  DeviceInfo di;
  cudaStream_t stream = nullptr, stream2 = nullptr;
  int pipe_min = 131072;  // records from which the memcpy path is split over two streams (env TSB200_PIPE_MIN)
  int pipe_chunk = 262144;
  uint8_t *d_in = nullptr, *d_out = nullptr;  // device chunk buffers (M_max records)
  uint8_t *h_in = nullptr, *h_out = nullptr;  // pinned+mapped staging, used when the caller's arrays cannot be locked
  size_t in_rec = 0, out_rec = 0;
  HostRegistry reg;
  int last_xfer = 0;  // TSB_XFER_ROUTE_* bits of the last host-buffer evaluate call
  uint64_t launches = 0;
  // fused expand (evaluate + generate_children on the device) and the device-resident pool
  ExpandCtx ex;
  uint8_t* d_children = nullptr;  // host-buffer expand: device image of the children
  size_t d_children_bytes = 0;
  DevicePool pool;
  RoundsCtx rounds;
  // Launch configuration of the handle's kernels, by kernel: the dynamic shared memory limit is raised on first use
  // (an attribute of the kernel in the device's context) and the CTAs per SM are queried once (0: not yet).
  struct KernelConfig {
    const void* fn;
    int per_sm;
  };
  std::vector<KernelConfig> kernels;

  int init(int dev, int M, size_t irec, size_t orec) {
    device = dev;
    M_max = M;
    in_rec = irec;
    out_rec = orec;
    xfer = env_xfer();
    int rc = query_device(dev, di);
    if (rc != TSB_OK) return rc;
    TSB_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    TSB_CUDA(cudaStreamCreateWithFlags(&stream2, cudaStreamNonBlocking));
    if (const char* v = std::getenv("TSB200_PIPE_MIN")) pipe_min = std::max(1, std::atoi(v));
    if (const char* v = std::getenv("TSB200_PIPE_CHUNK")) pipe_chunk = std::max(1024, std::atoi(v)) & ~1023;
    TSB_CUDA(cudaMalloc(&d_in, in_rec * M + 256));
    TSB_CUDA(cudaMalloc(&d_out, out_rec * M + 256));
    return TSB_OK;
  }
  int ensure_staging() {
    if (!h_in) TSB_CUDA(cudaHostAlloc(&h_in, in_rec * M_max + 256, cudaHostAllocPortable | cudaHostAllocMapped));
    if (!h_out) TSB_CUDA(cudaHostAlloc(&h_out, out_rec * M_max + 256, cudaHostAllocPortable | cudaHostAllocMapped));
    return TSB_OK;
  }
  void fini() {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    ex.release();
    rounds.release();
    if (d_children) cudaFree(d_children);
    pool.release();
    reg.release();
    if (d_in) cudaFree(d_in);
    if (d_out) cudaFree(d_out);
    if (h_in) cudaFreeHost(h_in);
    if (h_out) cudaFreeHost(h_out);
    if (bounce) cudaFreeHost(bounce);
    if (bounce_ev[0]) cudaEventDestroy(bounce_ev[0]);
    if (bounce_ev[1]) cudaEventDestroy(bounce_ev[1]);
    if (stream) cudaStreamDestroy(stream);
    if (stream2) cudaStreamDestroy(stream2);
  }

  // the kernel's launch configuration, with its dynamic shared memory limit raised to `smem`
  template <class K>
  int configure(K kernel, size_t smem, KernelConfig** cfg = nullptr) {
    const void* fn = reinterpret_cast<const void*>(kernel);
    KernelConfig* c = nullptr;
    for (KernelConfig& x : kernels)
      if (x.fn == fn) c = &x;
    if (!c) {
      TSB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
      kernels.push_back({fn, 0});
      c = &kernels.back();
    }
    if (cfg) *cfg = c;
    return TSB_OK;
  }
  // CTAs of `threads` threads and `smem` bytes of dynamic shared memory that one SM holds at once (at least 1)
  template <class K>
  int per_sm(K kernel, int threads, size_t smem, int* n) {
    KernelConfig* c = nullptr;
    int rc = configure(kernel, smem, &c);
    if (rc != TSB_OK) return rc;
    if (c->per_sm <= 0) {
      int blocks = 0;
      TSB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kernel, threads, smem));
      c->per_sm = std::max(blocks, 1);
    }
    *n = c->per_sm;
    return TSB_OK;
  }
  // persistent grid: enough CTAs to fill the GPU, never more than there are full tiles
  template <class K>
  int grid_for(K kernel, int threads, size_t smem, long long count, int tile, int* grid) {
    int n = 1;
    int rc = per_sm(kernel, threads, smem, &n);
    if (rc != TSB_OK) return rc;
    const long long tiles = std::max<long long>(1, count / tile);
    *grid = static_cast<int>(std::min<long long>(tiles, static_cast<long long>(n) * di.sms));
    return TSB_OK;
  }

  // What a finished launch of the persistent kernel `kernel` left in *st: TSB_ECUDA when its watchdog stopped it
  // (`stuck`: what did not complete); otherwise the pool [0, st->size) and the epoch are committed and
  // out[0..3] += {rounds, parents, children, solutions}.
  int finish_launch(const char* kernel, const char* stuck, tsb::RoundsState* st, uint64_t* out) {
    *st = *rounds.h_state;
    if (st->exit_code < 0 || st->exit_code == tsb::RND_EXIT_ABORT) {
      g_last_cuda_error = std::string(kernel) + ": watchdog abort (" + stuck + ")";
      return TSB_ECUDA;
    }
    rounds.epoch = st->epoch;
    pool.set_stack(st->size);
    out[0] += st->rounds;
    out[1] += st->parents;
    out[2] += st->children;
    out[3] += st->solutions;
    return TSB_OK;
  }

  // Copies between a caller-owned host range and the device, ordered on stream `s` (the stream the kernels
  // that produce / consume the data run on), synchronous.  Registered ranges are copied directly; anything else
  // bounces through two pinned buffers so that the host memcpy of one piece overlaps the DMA of the previous one.
  uint8_t* bounce = nullptr;
  cudaEvent_t bounce_ev[2] = {nullptr, nullptr};
  static constexpr size_t kBounce = 1 << 20;
  int ensure_bounce() {
    if (!bounce) {
      TSB_CUDA(cudaHostAlloc(&bounce, 2 * kBounce, cudaHostAllocPortable));
      TSB_CUDA(cudaEventCreateWithFlags(&bounce_ev[0], cudaEventDisableTiming));
      TSB_CUDA(cudaEventCreateWithFlags(&bounce_ev[1], cudaEventDisableTiming));
    }
    return TSB_OK;
  }
  int copy_h2d(void* dst_d, const void* src_h, size_t bytes, cudaStream_t s) {
    if (!bytes) return TSB_OK;
    if (reg.contains(src_h, bytes)) {
      TSB_CUDA(cudaMemcpyAsync(dst_d, src_h, bytes, cudaMemcpyHostToDevice, s));
      TSB_CUDA(cudaStreamSynchronize(s));
      return TSB_OK;
    }
    if (int rc = ensure_bounce(); rc != TSB_OK) return rc;
    int i = 0;
    for (size_t off = 0; off < bytes; off += kBounce, i++) {
      const size_t n = std::min(kBounce, bytes - off);
      uint8_t* b = bounce + (i & 1) * kBounce;
      if (i >= 2) TSB_CUDA(cudaEventSynchronize(bounce_ev[i & 1]));  // the DMA that last read this buffer is done
      std::memcpy(b, static_cast<const uint8_t*>(src_h) + off, n);
      TSB_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(dst_d) + off, b, n, cudaMemcpyHostToDevice, s));
      TSB_CUDA(cudaEventRecord(bounce_ev[i & 1], s));
    }
    TSB_CUDA(cudaStreamSynchronize(s));
    return TSB_OK;
  }
  int copy_d2h(void* dst_h, const void* src_d, size_t bytes, cudaStream_t s) {
    if (!bytes) return TSB_OK;
    if (reg.contains(dst_h, bytes)) {
      TSB_CUDA(cudaMemcpyAsync(dst_h, src_d, bytes, cudaMemcpyDeviceToHost, s));
      TSB_CUDA(cudaStreamSynchronize(s));
      return TSB_OK;
    }
    if (int rc = ensure_bounce(); rc != TSB_OK) return rc;
    const size_t pieces = (bytes + kBounce - 1) / kBounce;
    for (size_t i = 0; i <= pieces; i++) {  // DMA of piece i overlaps the host memcpy of piece i-1
      if (i < pieces) {
        const size_t off = i * kBounce, n = std::min(kBounce, bytes - off);
        TSB_CUDA(cudaMemcpyAsync(bounce + (i & 1) * kBounce, static_cast<const uint8_t*>(src_d) + off, n,
                                 cudaMemcpyDeviceToHost, s));
        TSB_CUDA(cudaEventRecord(bounce_ev[i & 1], s));
      }
      if (i >= 1) {
        const size_t off = (i - 1) * kBounce, n = std::min(kBounce, bytes - off);
        TSB_CUDA(cudaEventSynchronize(bounce_ev[(i - 1) & 1]));
        std::memcpy(static_cast<uint8_t*>(dst_h) + off, bounce + ((i - 1) & 1) * kBounce, n);
      }
    }
    return TSB_OK;
  }

  // Host-buffer evaluation shared by N-Queens and PFSP.  `launch(in_dev, out_dev, count, stream)`
  // enqueues the evaluator kernel.
  template <class Launch>
  int evaluate_host(const void* in, int count, void* out, Launch&& launch) {
    const size_t in_b = in_rec * count, out_b = out_rec * count;
    const bool in_locked = reg.contains(in, in_b), out_locked = reg.contains(out, out_b);
    // AUTO: zero-copy whenever the caller registered its arrays (tsb_*_register_host) and they are 16-byte
    // aligned (fastest at every chunk size in tools/xfer_sweep.py's comparison); otherwise copies, pipelined
    // when large, through the handle's pinned staging buffers for arrays that are not registered
    last_xfer = tsb::xfer_route(xfer, in_locked, out_locked, reinterpret_cast<uintptr_t>(in),
                                reinterpret_cast<uintptr_t>(out), di.can_use_host_ptr, count, pipe_min, pipe_chunk);

    if (last_xfer & TSB_XFER_ROUTE_ZEROCOPY) {
      // the kernel's TMA engine pulls the chunk over PCIe and pushes the results back: one launch,
      // reads and writes overlap on the full-duplex link
      int rc = launch(static_cast<const uint8_t*>(in), static_cast<uint8_t*>(out), count, stream);
      if (rc != TSB_OK) return rc;
      TSB_CUDA(cudaStreamSynchronize(stream));
      return TSB_OK;
    }
    const uint8_t* src = static_cast<const uint8_t*>(in);
    uint8_t* dst = static_cast<uint8_t*>(out);
    if (!in_locked || !out_locked) {
      int rc = ensure_staging();
      if (rc != TSB_OK) return rc;
    }
    if (!in_locked) src = h_in;
    if (!out_locked) dst = h_out;
    if (last_xfer & TSB_XFER_ROUTE_PIPELINED) {
      // large chunk: sub-chunks alternate between two streams so that the upload of one overlaps the
      // download of the previous one (PCIe is full duplex) and the kernel of the one in between; the host
      // memcpy into the staging buffer of sub-chunk i+1 overlaps the device work of sub-chunk i
      const cudaStream_t st[2] = {stream, stream2};
      int i = 0;
      for (int off = 0; off < count; off += pipe_chunk, ++i) {
        const int n = std::min(pipe_chunk, count - off);
        cudaStream_t s = st[i & 1];
        if (!in_locked) std::memcpy(h_in + in_rec * off, static_cast<const uint8_t*>(in) + in_rec * off, in_rec * n);
        TSB_CUDA(cudaMemcpyAsync(d_in + in_rec * off, src + in_rec * off, in_rec * n, cudaMemcpyHostToDevice, s));
        int rc = launch(d_in + in_rec * off, d_out + out_rec * off, n, s);
        if (rc != TSB_OK) return rc;
        TSB_CUDA(cudaMemcpyAsync(dst + out_rec * off, d_out + out_rec * off, out_rec * n, cudaMemcpyDeviceToHost, s));
      }
      TSB_CUDA(cudaStreamSynchronize(stream));
      TSB_CUDA(cudaStreamSynchronize(stream2));
    } else {
      if (!in_locked) std::memcpy(h_in, in, in_b);
      TSB_CUDA(cudaMemcpyAsync(d_in, src, in_b, cudaMemcpyHostToDevice, stream));
      int rc = launch(d_in, d_out, count, stream);
      if (rc != TSB_OK) return rc;
      TSB_CUDA(cudaMemcpyAsync(dst, d_out, out_b, cudaMemcpyDeviceToHost, stream));
      TSB_CUDA(cudaStreamSynchronize(stream));
    }
    if (!out_locked) std::memcpy(out, h_out, out_b);
    return TSB_OK;
  }
};

// f(std::integral_constant<int, N>) for the board size N = 1..MAXN
template <int N = 1, int MAXN = TSB_MAX_QUEENS, class F>
int with_queens(int n, F&& f) {
  if constexpr (N > MAXN)
    return TSB_EINVAL;
  else
    return n == N ? f(std::integral_constant<int, N>{}) : with_queens<N + 1, MAXN>(n, f);
}
// f(std::integral_constant<int, M>) for the template machine count mt = 5, 10 or 20
template <class F>
int with_machines(int mt, F&& f) {
  if (mt == 5) return f(std::integral_constant<int, 5>{});
  if (mt == 10) return f(std::integral_constant<int, 10>{});
  return f(std::integral_constant<int, 20>{});
}

// bounds are int32 and `lb > best` can never hold for best >= INT32_MAX (Chapel's max(int) under --ub 0)
inline int clamp_best(int64_t best64) {
  return best64 > INT_MAX ? INT_MAX : best64 < INT_MIN ? INT_MIN : static_cast<int>(best64);
}

// tile table of a round: pieces in logical order -> ExpandParams
int make_params(const std::vector<PoolExtent>& pieces, int tile_records, tsb::ExpandParams* prm) {
  if (pieces.empty() || pieces.size() > tsb::EXP_MAX_PIECES) return TSB_EINVAL;
  std::memset(prm, 0, sizeof(*prm));
  long long cum = 0;
  for (size_t i = 0; i < pieces.size(); i++) {
    const PoolExtent& x = pieces[i];
    const long long t0 = x.b / tile_records, t1 = (x.e + tile_records - 1) / tile_records;
    prm->piece[i].lo = x.b;
    prm->piece[i].hi = x.e;
    prm->piece[i].first_tile = t0;
    prm->piece[i].tile_cum = static_cast<int>(cum);
    cum += t1 - t0;
  }
  if (cum > INT_MAX / 2) return TSB_EINVAL;
  prm->n_pieces = static_cast<int>(pieces.size());
  prm->n_tiles = static_cast<int>(cum);
  return TSB_OK;
}

// ---- device-pool operations of both handle types.  `plain()` brings the pool into its plain arena first (the
// N-Queens pool may live in the persistent kernel's own format); `expand(arena, pieces, children_d, &nc, &ns)` runs
// one evaluate + generate_children round on the handle's stream.

template <class Plain>
int pool_push(Base& h, const void* nodes, int64_t n, Plain&& plain) {
  TSB_CUDA(cudaSetDevice(h.device));
  int rc = plain();
  if (rc != TSB_OK) return rc;
  DevicePool& p = h.pool;
  rc = p.reserve(h.stream, n);
  if (rc != TSB_OK) return rc;
  if (n == 0) return TSB_OK;
  const long long at = p.top();
  // (on the handle's non-blocking stream, which the kernels of the next round are ordered after)
  rc = h.copy_h2d(p.arena[p.cur] + at * p.rec, nodes, static_cast<size_t>(n) * p.rec, h.stream);
  if (rc != TSB_OK) return rc;
  if (p.ext.empty())
    p.ext.push_back({at, at + n});
  else
    p.ext.back().e += n;
  p.size += n;
  return TSB_OK;
}

template <class Plain>
int pool_drain(Base& h, void* nodes, int64_t capacity, int64_t* n, Plain&& plain) {
  DevicePool& p = h.pool;
  *n = p.size;
  if (p.size > capacity) return TSB_ENOMEM;
  TSB_CUDA(cudaSetDevice(h.device));
  if (int rc = plain(); rc != TSB_OK) return rc;
  long long at = 0;
  for (const PoolExtent& x : p.ext) {  // extents are the pool in logical (oldest first) order
    int rc = h.copy_d2h(static_cast<uint8_t*>(nodes) + at * p.rec, p.arena[p.cur] + x.b * p.rec,
                        static_cast<size_t>(x.e - x.b) * p.rec, h.stream);
    if (rc != TSB_OK) return rc;
    at += x.e - x.b;
  }
  p.ext.clear();
  p.size = 0;
  return TSB_OK;
}

// one round: popBackBulk(m, M), expand, the children pushed
template <class Plain, class Expand>
int pool_step(Base& h, int m, int M, int64_t* n_parents, uint64_t* n_children, uint64_t* n_solutions, Plain&& plain,
              Expand&& expand) {
  *n_parents = 0;
  *n_children = *n_solutions = 0;
  DevicePool& p = h.pool;
  if (p.size < m) return TSB_OK;  // popBackBulk returns 0 below m (lib/commons/Pool.chpl:50-59)
  TSB_CUDA(cudaSetDevice(h.device));
  int rc = plain();
  if (rc != TSB_OK) return rc;
  const long long n = std::min<long long>(p.size, M);
  // room above the top for the worst case (every slot of every parent survives) and the children's alignment; the
  // chunk itself is read in place, as the newest pieces of the extent stack
  std::vector<PoolExtent> pieces;
  p.top_pieces(n, &pieces);
  if (pieces.size() > tsb::EXP_MAX_PIECES) rc = p.compact(h.stream, p.cap);
  if (rc == TSB_OK) rc = p.reserve(h.stream, n * p.fanout + 2 * (p.align - 1));
  if (rc != TSB_OK) return rc;
  p.top_pieces(n, &pieces);  // (positions change when the pool was compacted)
  const long long top = p.aligned_top();
  unsigned long long nc = 0, ns = 0;
  uint8_t* arena = p.arena[p.cur];
  rc = expand(arena, pieces, arena + top * p.rec, &nc, &ns);
  if (rc != TSB_OK) return rc;
  p.pop(n);
  p.push_extent(top, static_cast<long long>(nc));
  *n_parents = n;
  *n_children = nc;
  *n_solutions = ns;
  return TSB_OK;
}

// `step(&np, &nc, &ns)` until a round takes no parents or max_rounds rounds have run; out[] += {rounds, parents,
// children, solutions}
template <class Step>
int step_loop(int64_t max_rounds, uint64_t* out, Step&& step) {
  for (int64_t r = 0; r < max_rounds; r++) {
    int64_t np = 0;
    uint64_t nc = 0, ns = 0;
    const int rc = step(&np, &nc, &ns);
    if (rc != TSB_OK) return rc;
    if (np == 0) break;
    out[0] += 1;
    out[1] += static_cast<uint64_t>(np);
    out[2] += nc;
    out[3] += ns;
  }
  return TSB_OK;
}

// ---- the persistent kernel's host loop, over a problem type R (NqRounds, PfspRounds) that supplies the handle, sync
// and parameter types and: grid(h0, M, pools, &variant) (CTAs per pool, 0: the launch does not take M);
// prepare(h, i, left, need, &prm, &queued) (pool i's arena ready for a next round of up to `need` nodes, prm's own
// fields; queued: work on h's stream the launch must follow); launch(h0, params, grid, pools, variant) on h0's stream;
// resume(h, i, st, m, M, &left, out, &again) (what pool i does after its exit code); step (one two-kernel round of
// pool i); report (the TSB200_ROUNDS_PROF lines of a launch); of_pool(i) (pool i's problem on its own).

// Up to max_rounds rounds of EACH of the K pools hs[0..K) (handles on one device) in launches of R's persistent kernel
// that serve every pool that still has work: grid (G, pools).  out[4 i ..] += {rounds, parents, children, solutions}
// of pool i.  A pool leaves a launch on its own: when it holds fewer than m nodes, after its round budget, when its
// next round's worst case does not fit its arena (it grows and goes again), or for a reason of R's (R::resume).  The
// launch ends when every pool has left; the grid follows the number of pools that still run.
template <class R>
int rounds_run(const R& r, typename R::Handle* const* hs, int K, int m, int M, int64_t max_rounds, uint64_t* out) {
  int64_t left[R::kMaxPools];
  bool active[R::kMaxPools];
  for (int i = 0; i < K; i++) {
    left[i] = max_rounds;
    active[i] = true;
  }
  const bool prof = std::getenv("TSB200_ROUNDS_PROF") != nullptr;
  for (;;) {
    int map[R::kMaxPools], n_act = 0;
    for (int i = 0; i < K; i++) {
      active[i] = active[i] && hs[i]->pool.size >= m && left[i] > 0;
      if (active[i]) map[n_act++] = i;
    }
    if (n_act == 0) return TSB_OK;
    typename R::Handle* h0 = hs[map[0]];
    int variant = 0;
    const int grid = r.grid(h0, M, n_act, &variant);
    if (grid == 0) {
      // A launch that takes K >= 2 pools takes any 2..K of them (the callers check K), but one pool alone may not be
      // taken at the same M: the one-pool kernel has a smaller capacity (ll_tiers.h) or a lower limit (PFR_MAX_M).
      // The last pool then finishes in two-kernel rounds, as pool_run runs it.
      if (n_act > 1) return TSB_EINVAL;
      const int i = map[0];
      return step_loop(left[i], &out[4 * i], [&](int64_t* np, uint64_t* nc, uint64_t* ns) {
        return r.step(h0, i, m, M, np, nc, ns);
      });
    }
    typename R::Params mp;
    std::memset(&mp, 0, sizeof(mp));
    long long need[R::kMaxPools];
    for (int a = 0; a < n_act; a++) {
      const int i = map[a];
      typename R::Handle* h = hs[i];
      const long long n = std::min<long long>(h->pool.size, M);
      need[a] = h->pool.size - n + n * h->pool.fanout;  // the worst case of the next round
      bool queued = !h->rounds.d_sync;  // (a new handle's flags are cleared on its stream)
      int rc = h->rounds.template ensure<typename R::Sync>(h->stream);
      if (rc == TSB_OK) rc = r.prepare(h, i, left[i], need[a], &mp.pool[a], &queued);
      if (rc != TSB_OK) return rc;
      if (queued && a > 0) TSB_CUDA(cudaStreamSynchronize(h->stream));  // (the launch goes on the first pool's stream)
      auto& prm = mp.pool[a];
      prm.size0 = h->pool.size;
      prm.epoch0 = h->rounds.epoch;
      prm.m = m;
      prm.M = M;
      prm.max_rounds = left[i];
      prm.prof = prof;
      prm.sync = h->rounds.template sync<typename R::Sync>();
      prm.state = h->rounds.d_state;
      h->rounds.h_state->exit_code = -1;
    }
    int rc = r.launch(h0, mp, grid, n_act, variant);
    if (rc != TSB_OK) return rc;
    TSB_CUDA(cudaStreamSynchronize(h0->stream));
    tsb::RoundsState st[R::kMaxPools];
    for (int a = 0; a < n_act; a++) {
      const int i = map[a];
      typename R::Handle* h = hs[i];
      rc = h->finish_launch(R::kKernel, R::kStuck, &st[a], &out[4 * i]);
      if (rc != TSB_OK) return rc;
      left[i] -= static_cast<int64_t>(st[a].rounds);
      if (st[a].exit_code == tsb::RND_EXIT_SPACE && st[a].rounds == 0 && need[a] <= h->pool.cap)
        return TSB_ENOMEM;  // (cannot happen: the arena was grown for `need`)
      rc = r.resume(h, i, st[a], m, M, &left[i], &out[4 * i], &active[i]);
      if (rc != TSB_OK) return rc;
    }
    if (prof) r.report(st, map, n_act, grid);
  }
}

// one pool: the persistent kernel when it takes M, else two-kernel rounds
template <class R>
int pool_run(const R& r, typename R::Handle* h, int m, int M, int64_t max_rounds, uint64_t* n_rounds,
             uint64_t* n_parents, uint64_t* n_children, uint64_t* n_solutions) {
  *n_rounds = *n_parents = *n_children = *n_solutions = 0;
  TSB_CUDA(cudaSetDevice(h->device));
  uint64_t out[4] = {0, 0, 0, 0};
  const int rc = rounds_run(r, &h, 1, m, M, max_rounds, out);
  *n_rounds = out[0];
  *n_parents = out[1];
  *n_children = out[2];
  *n_solutions = out[3];
  return rc;
}

// K pools in shared launches, or one pool after the other when one launch does not take K pools at this M
template <class R>
int pool_run_multi(const R& r, typename R::Handle* const* hs, int K, int m, int M, int64_t max_rounds, uint64_t* out) {
  std::memset(out, 0, sizeof(uint64_t) * 4 * K);
  TSB_CUDA(cudaSetDevice(hs[0]->device));
  if (r.grid(hs[0], M, K, nullptr) > 0) return rounds_run(r, hs, K, m, M, max_rounds, out);
  for (int i = 0; i < K; i++) {
    const int rc = rounds_run(r.of_pool(i), &hs[i], 1, m, M, max_rounds, &out[4 * i]);
    if (rc != TSB_OK) return rc;
  }
  return TSB_OK;
}

// the most pools one launch takes with chunks of up to M parents (1: not several)
template <class R, class H>
int pools_per_launch(const R& r, H* h, int M) {
  for (int pools = R::kMaxPools; pools > 1; pools--)
    if (r.grid(h, M, pools, nullptr) > 0) return pools;
  return 1;
}

// expand of host arrays: the parents through d_in, the children through d_children (room for M_max parents' worst
// case)
template <class Expand>
int expand_host(Base& h, const void* parents, int count, void* children, uint64_t capacity, uint64_t* n_children,
                uint64_t* n_solutions, Expand&& expand) {
  TSB_CUDA(cudaSetDevice(h.device));
  const size_t rec = h.pool.rec, need = static_cast<size_t>(h.M_max) * h.pool.fanout * rec + 64;
  if (h.d_children_bytes < need) {
    if (h.d_children) cudaFree(h.d_children);
    h.d_children = nullptr;
    h.d_children_bytes = 0;
    TSB_CUDA(cudaMalloc(&h.d_children, need));
    h.d_children_bytes = need;
  }
  int rc = h.copy_h2d(h.d_in, parents, rec * static_cast<size_t>(count), h.stream);
  if (rc != TSB_OK) return rc;
  unsigned long long nc = 0, ns = 0;
  const std::vector<PoolExtent> pieces{{0, count}};
  rc = expand(h.d_in, pieces, h.d_children, &nc, &ns);
  if (rc != TSB_OK) return rc;
  *n_children = nc;
  *n_solutions = ns;
  if (nc > capacity) return TSB_ENOMEM;  // the caller's children array is too small; counts are valid
  return h.copy_d2h(children, h.d_children, nc * rec, h.stream);
}

// Work stealing between device pools (SURVEY §8f row 3; the reference steals between its per-GPU host pools,
// nqueens_multigpu_chpl.chpl:255-312): the OLDEST half of the victim's pool (popFrontBulkFree,
// lib/commons/Pool_par.chpl:178-191: size / 2 nodes from the front, only if size >= 2 m) moves to the top of the
// thief's pool, device to device (cudaMemcpyPeerAsync: peer-to-peer between two GPUs, a plain copy on one), order
// preserved.  Both pools must be quiescent (no round in flight); the caller serialises access to both handles.
// `plain()` brings both pools into their plain arenas.
template <class Plain>
int pool_steal(Base& victim, Base& thief, int m, int64_t* n_stolen, Plain&& plain) {
  *n_stolen = 0;
  DevicePool &v = victim.pool, &t = thief.pool;
  if (v.size < 2LL * m) return TSB_OK;
  int rc = plain();
  if (rc != TSB_OK) return rc;
  const long long want = v.size / 2;
  const bool trace = std::getenv("TSB200_TRACE") != nullptr;
  const auto tnow = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double tr0 = trace ? tnow() : 0;
  TSB_CUDA(cudaSetDevice(thief.device));
  rc = t.reserve(thief.stream, want);
  if (rc != TSB_OK) return rc;
  long long at = t.aligned_top();
  if (at + want > t.cap) {
    rc = t.compact(thief.stream, std::max<long long>(2 * t.cap, t.size + want + 1024));
    if (rc != TSB_OK) return rc;
    at = t.aligned_top();
  }
  TSB_CUDA(cudaSetDevice(victim.device));
  long long left = want, dst = at;
  while (left > 0 && !v.ext.empty()) {
    PoolExtent& x = v.ext.front();
    const long long n = std::min(left, x.e - x.b);
    TSB_CUDA(cudaMemcpyPeerAsync(t.arena[t.cur] + dst * t.rec, thief.device, v.arena[v.cur] + x.b * v.rec,
                                 victim.device, static_cast<size_t>(n) * v.rec, victim.stream));
    x.b += n;
    dst += n;
    left -= n;
    if (x.b == x.e) v.ext.erase(v.ext.begin());
  }
  TSB_CUDA(cudaStreamSynchronize(victim.stream));
  const long long got = want - left;
  v.size -= got;
  t.push_extent(at, got);
  *n_stolen = got;
  if (trace)
    std::fprintf(stderr, "[tsb200] steal: %lld nodes (%.1f MB) device %d -> %d in %.2f ms (victim keeps %lld, thief has %lld)\n",
                 got, got * v.rec / 1e6, victim.device, thief.device, tnow() - tr0, v.size, t.size);
  return TSB_OK;
}

// Everything the kernels of a PFSP handle read, packed once from the tsb_pfsp_create arguments: a handle and its
// siblings share one immutable copy, so a sibling takes its owner's route as it was fixed at creation
struct PfspPacked {
  int jobs = 0, machines = 0;
  int pairs = 0;         // 0: no lb2 on this handle
  int mt = 0;            // template machine count (5, 10 or 20)
  bool wide = false;     // MAX_JOBS = 50: 208-byte nodes, the general kernels of pfsp_wide.cuh
  bool simd16 = false;   // lb1 / lb1_d children two per register (values < 2^16, min_tails non-increasing)
  bool lb2u = false;     // <= 10 machines: lb2 on the shared-memory-resident table `tabu`
  bool valid = true;     // every machine pair, mp_order and Johnson index in range
  tsb::PfspLb1Tables t1;   // 20 jobs
  tsb::PfspWideTables tw;  // 50 jobs (lb2 tables included)
  tsb::Lb2Const lb2c;      // 20 jobs: packed Johnson tables, passed to the lb2 kernels by value (constant bank)
  tsb::Lb2TabU tabu;
};

// The tables for the reference built with MAX_JOBS = max_jobs (20 or 50), from arguments whose pointers and shape
// tsb_pfsp_create_wide has checked.  Indices out of range clear `valid`; values that do not fit the lb2 words leave
// the handle without lb2.  TSB200_NO_SIMD16 / TSB200_NO_LB2U (any value but "0" for the latter) turn routes off.
std::shared_ptr<const PfspPacked> pfsp_pack(int max_jobs, int jobs, int machines, const int32_t* p_times,
                                            const int32_t* min_heads, const int32_t* min_tails, int nb_pairs,
                                            const int32_t* johnson, const int32_t* lags, const int32_t* mp0,
                                            const int32_t* mp1, const int32_t* mp_order) {
  auto t = std::make_shared<PfspPacked>();  // (value-initialised: every table and its padding start at zero)
  t->jobs = jobs;
  t->machines = machines;
  t->pairs = nb_pairs;
  t->mt = machines <= 5 ? 5 : machines <= 10 ? 10 : 20;
  t->wide = max_jobs != TSB_MAX_JOBS;
  tsb::PfspLb1Tables& t1 = t->t1;
  tsb::PfspWideTables& tw = t->tw;
  t1.jobs = tw.jobs = jobs;
  t1.machines = tw.machines = machines;
  t1.pairs = tw.pairs = nb_pairs;
  t1.mp = tsb::row_stride(t->mt);
  // lb1 (zero padding up to the template machine count is value-neutral: the reference itself evaluates 20-wide
  // zero-padded tuples, lib/pfsp/Bound_simple.chpl:125-135)
  int32_t* total = t->wide ? tw.total : t1.total;
  int32_t* pj = t->wide ? tw.pj : t1.pj;
  const int mp = t->wide ? tsb::PW_PSTRIDE : t1.mp, hs = tsb::half_stride(t->mt);
  long long sum_all = 0, max_head = 0, max_tail = 0;
  bool nonneg = true, tails_monotone = true;
  for (int k = 0; k < machines; k++) {
    (t->wide ? tw.min_heads : t1.min_heads)[k] = min_heads[k];
    (t->wide ? tw.min_tails : t1.min_tails)[k] = min_tails[k];
    max_head = std::max<long long>(max_head, min_heads[k]);
    max_tail = std::max<long long>(max_tail, min_tails[k]);
    nonneg &= min_heads[k] >= 0 && min_tails[k] >= 0;
    if (k > 0) tails_monotone &= min_tails[k] <= min_tails[k - 1];
    for (int j = 0; j < jobs; j++) {
      const int32_t pv = p_times[k * jobs + j];
      total[k] += pv;
      pj[j * mp + k] = pv;
      nonneg &= pv >= 0;
      sum_all += pv;
      if (!t->wide) t1.ph[j * hs + (k >> 1)] |= static_cast<uint32_t>(pv & 0xFFFF) << (16 * (k & 1));
    }
  }
  // every intermediate of the bounds is <= sum of all processing times + largest head + largest tail
  t->simd16 = !t->wide && nonneg && tails_monotone && sum_all + max_head + max_tail < tsb::PF_LANE_LIMIT &&
              !std::getenv("TSB200_NO_SIMD16");
  // lb2: Johnson tables in machine_pair_order
  const uint32_t lag_max = t->wide ? tsb::PW_LAG_MAX : tsb::LB2_LAG_MAX;
  bool fits = true;
  for (int l = 0; l < nb_pairs; l++) {
    const int i = mp_order[l];
    if (i < 0 || i >= nb_pairs) {
      t->valid = false;
      continue;
    }
    const int a = mp0[i], b = mp1[i];
    if (a < 0 || a >= machines || b < 0 || b >= machines) {
      t->valid = false;
      continue;
    }
    fits &= tsb::lb2_fits(min_tails[a], tsb::LB2_TAIL_MAX) && tsb::lb2_fits(min_tails[b], tsb::LB2_TAIL_MAX);
    (t->wide ? tw.pair : t->lb2c.pair)[l] = tsb::lb2_pair_word(a, b, min_tails[a], min_tails[b]);
    for (int j = 0; j < jobs; j++) {
      const int job = johnson[i * jobs + j];
      if (job < 0 || job >= jobs) {
        t->valid = false;
        continue;
      }
      const int pa = p_times[a * jobs + job], pb = p_times[b * jobs + job], lg = lags[i * jobs + job];
      fits &= tsb::lb2_fits(pa, tsb::LB2_P_MAX) && tsb::lb2_fits(pb, tsb::LB2_P_MAX) && tsb::lb2_fits(lg, lag_max);
      if (t->wide)
        tw.jp[l * jobs + j] = tsb::pw_job_word(job, pa, pb, lg);
      else
        t->lb2c.jp[l * tsb::PF_MAXJ + j] = tsb::lb2_job_word(job, pa, pb, lg);
    }
  }
  if (!fits) t->pairs = 0;  // values outside the Taillard range: no lb2 on this handle
  const char* no_u = std::getenv("TSB200_NO_LB2U");
  t->lb2u = t->valid && t->pairs > 0 && nb_pairs <= tsb::LB2U_PAIRS && t->mt <= 10 && t->simd16 &&
            !(no_u && *no_u && *no_u != '0');
  for (int l = 0; l < nb_pairs && t->lb2u; l++) {
    const int i = mp_order[l], a = mp0[i], b = mp1[i];
    t->tabu.mach[l] = tsb::lb2u_mach_word(a, b);
    t->tabu.tails[l] = tsb::lb2u_tails_word(min_tails[a], min_tails[b]);
    for (int j = 0; j < jobs; j++) {
      const int job = johnson[i * jobs + j];
      t->tabu.e[l * tsb::PF_MAXJ + j] = tsb::lb2u_entry(job, p_times[a * jobs + job], p_times[b * jobs + job],
                                                        lags[i * jobs + job]);
    }
  }
  return t;
}

// handle-level entry points of both handle types
int register_host(Base* h, void* ptr, size_t bytes) {
  if (!h) return TSB_EINVAL;
  TSB_CUDA(cudaSetDevice(h->device));
  return h->reg.add(ptr, bytes);
}
int unregister_host(Base* h, void* ptr) {
  if (!h) return TSB_EINVAL;
  TSB_CUDA(cudaSetDevice(h->device));
  return h->reg.remove(ptr);
}
int set_xfer(Base* h, int mode) {
  if (!h || mode < 0 || mode > 2) return TSB_EINVAL;
  h->xfer = mode;
  return TSB_OK;
}
int last_xfer(const Base* h) { return h ? h->last_xfer : TSB_EINVAL; }
void* stream_of(const Base* h) { return h ? static_cast<void*>(h->stream) : nullptr; }
int64_t pool_size(const Base* h) { return h ? h->pool.size : -1; }

// the handle and the siblings it owns; each handle type frees its own device buffers in its destructor
template <class H>
void destroy(H* h) {
  if (!h) return;
  for (H*& x : h->sibling) {
    destroy(x);
    x = nullptr;
  }
  h->fini();
  delete h;
}

// launches of the handle and of its siblings
template <class H>
uint64_t kernel_launches(const H* h) {
  if (!h) return 0;
  uint64_t n = h->launches;
  for (const H* x : h->sibling)
    if (x) n += x->launches;
  return n;
}

// sibling `index` (1..3) of h, created by make(&slot) on first use and owned by h
template <class H, class Make>
int sibling_of(H* h, int index, H** sibling, Make&& make) {
  if (!h || !sibling || index < 1 || index > static_cast<int>(std::size(h->sibling))) return TSB_EINVAL;
  H*& s = h->sibling[index - 1];
  if (!s)
    if (const int rc = make(&s); rc != TSB_OK) return rc;
  *sibling = s;
  return TSB_OK;
}

// the pools of one tsb_*_pool_run_multi call: distinct handles of one kind (`same(h, h0)`) on one device, each
// taking chunks of M parents
template <class H, class Same>
bool one_group(H* const* hs, int K, int M, Same&& same) {
  for (int i = 0; i < K; i++) {
    const H* h = hs[i];
    if (!h || M > h->M_max || h->device != hs[0]->device || !same(*h, *hs[0])) return false;
    for (int j = 0; j < i; j++)
      if (hs[j] == h) return false;
  }
  return true;
}

void enable_peer(int a, int b) {
  if (a == b) return;
  int can = 0;
  if (cudaDeviceCanAccessPeer(&can, a, b) == cudaSuccess && can) {
    cudaSetDevice(a);
    if (cudaDeviceEnablePeerAccess(b, 0) != cudaSuccess) (void)cudaGetLastError();  // (already enabled is fine)
  }
  (void)cudaGetLastError();
}

}  // namespace

// ============================================================================ handles
struct tsb_nq : Base {
  ~tsb_nq() {
    if (d_fat) cudaFree(d_fat);
  }
  tsb_nq* sibling[3] = {nullptr, nullptr, nullptr};  // further pools on the same device, owned by this handle (tsb_nq_sibling)
  int N = 0, g = 1;
  bool wide = false;  // MAX_QUEENS = 24 build (tsb_nq_create_wide): 25-byte tsb_nq_node24 records, one pool per launch
  int tile_threads = 0;  // env TSB200_NQ_TILE_THREADS = 128: always the TMA-pipelined kernel (tests force it on small chunks)
  tsb::FatNode* d_fat = nullptr;  // the pool in the self-validating 32-byte format, while the LL kernel owns it
  long long fat_cap = 0;
  bool in_fat = false;  // the pool currently lives in d_fat (the plain arena is stale)
  // 16-bit tags of d_fat (nq_rounds_ll.cuh): the epoch of its last clear, and the highest pool size since then (every
  // word at or above it carries tag 0)
  unsigned tag_clear = 0;
  long long tag_hi = 0;
};

struct tsb_pfsp : Base {
  ~tsb_pfsp() {
    if (d_tab1) cudaFree(d_tab1);
    if (d_wtab) cudaFree(d_wtab);
    if (d_tabu) cudaFree(d_tabu);
  }
  tsb_pfsp* sibling[3] = {nullptr, nullptr, nullptr};  // further pools on the same device, owned by this handle (tsb_pfsp_sibling)
  std::shared_ptr<const PfspPacked> tab;  // the tables and route, shared with the owner or the siblings
  // device copies of tab's tables: t1 or tw, and tabu on the lb2u route
  tsb::PfspLb1Tables* d_tab1 = nullptr;
  tsb::PfspWideTables* d_wtab = nullptr;
  tsb::Lb2TabU* d_tabu = nullptr;
  uint64_t slow_rounds = 0;
  std::vector<tsb_pfsp_node> h_chunk, h_kids;  // slow path scratch
  std::vector<tsb_pfsp_node50> h_chunk50, h_kids50;
  std::vector<int32_t> h_bounds;
};

namespace {

// ============================================================================ N-Queens
// f(std::integral_constant<int, N>, std::integral_constant<int, R>) for the handle's board size N and record width R
template <class F>
int with_board(const tsb_nq* h, F&& f) {
  if (h->wide)
    return with_queens<1, TSB_MAX_QUEENS_WIDE>(h->N, [&](auto n) { return f(n, std::integral_constant<int, tsb::NQ_REC24>{}); });
  return with_queens(h->N, [&](auto n) { return f(n, std::integral_constant<int, tsb::NQ_REC>{}); });
}

// small chunks (fewer than two 512-parent tiles per SM — the reference's default --M 50000 is 97 tiles) take the
// one-parent-per-thread kernel, everything else the TMA-pipelined one
template <int N, int R>
int launch_nq_n(tsb_nq* h, const uint8_t* in, uint8_t* out, long long count, cudaStream_t s) {
  if (count < 2LL * h->di.sms * tsb::NQ_TILE && h->tile_threads != 128) {
    const int grid = static_cast<int>((count + tsb::NQ_SMALL - 1) / tsb::NQ_SMALL);
    tsb::NqKernels<N, R>::evaluate_small<<<grid, tsb::NQ_SMALL, 0, s>>>(in, out, static_cast<int>(count));
    TSB_CUDA(cudaGetLastError());
    h->launches++;
    return TSB_OK;
  }
  auto kernel = tsb::NqKernels<N, R>::evaluate;
  const size_t smem = sizeof(tsb::NqSmem<N, R>) + 128;
  int grid = 1;
  int rc = h->grid_for(kernel, tsb::NQ_THREADS, smem, count, tsb::NQ_TILE, &grid);
  if (rc != TSB_OK) return rc;
  kernel<<<grid, tsb::NQ_THREADS, smem, s>>>(in, out, count);
  TSB_CUDA(cudaGetLastError());
  h->launches++;
  return TSB_OK;
}

int launch_nq(tsb_nq* h, const uint8_t* in, uint8_t* out, long long count, cudaStream_t s) {
  return with_board(h, [&](auto n, auto r) { return launch_nq_n<decltype(n)::value, decltype(r)::value>(h, in, out, count, s); });
}

// one evaluate + generate_children round over `pieces` of `arena` (count, build); children packed at
// `children_d`.  Synchronous: the counts come back through the host-mapped result record.
template <int N, int R>
int nq_expand_n(tsb_nq* h, const uint8_t* arena, const std::vector<PoolExtent>& pieces, uint8_t* children_d,
                cudaStream_t s, unsigned long long* n_children, unsigned long long* n_solutions, bool early) {
  tsb::ExpandParams prm;
  int rc = make_params(pieces, tsb::NQ_TILE, &prm);
  if (rc != TSB_OK) return rc;
  ExpandCtx& ex = h->ex;
  const bool trace = ex.epoch == 0 && std::getenv("TSB200_TRACE");  // (the handle's first round)
  const auto tnow = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double tr0 = trace ? tnow() : 0;
  // (sized for the largest round up front: the items array is 1 KB * N per tile)
  rc = ex.reserve(std::max<long long>(prm.n_tiles, h->M_max / tsb::NQ_TILE + 2 * tsb::EXP_MAX_PIECES),
                  static_cast<long long>(tsb::NQ_TILE) * N * 2, s);
  if (rc != TSB_OK) return rc;
  auto k1 = tsb::NqKernels<N, R>::count;
  auto k3 = tsb::NqKernels<N, R>::build;
  const size_t smem1 = sizeof(tsb::NqCountSmem<R>) + 128, smem3 = sizeof(tsb::NqBuildSmem<R>) + 128;
  const long long recs = static_cast<long long>(prm.n_tiles) * tsb::NQ_TILE;
  int g1 = 1, g3 = 1;
  rc = h->grid_for(k1, tsb::NQ_THREADS, smem1, recs, tsb::NQ_TILE, &g1);
  if (rc != TSB_OK) return rc;
  rc = h->grid_for(k3, tsb::NQ_THREADS, smem3, recs, tsb::NQ_TILE, &g3);
  if (rc != TSB_OK) return rc;
  prm.epoch = ++ex.epoch;
  if ((prm.n_tiles + g3 - 1) / g3 > tsb::EXP_MAX_OWN) return TSB_EINVAL;  // (M_max * N < 2^31 keeps this far away)
  uint16_t* d_items = reinterpret_cast<uint16_t*>(ex.d_cmask);
  const double tr1 = trace ? tnow() : 0;
  k1<<<g1, tsb::NQ_THREADS, smem1, s>>>(arena, prm, d_items, ex.d_tile, ex.d_st);
  k3<<<g3, tsb::NQ_THREADS, smem3, s>>>(arena, prm, d_items, ex.d_tile, children_d, ex.d_st, ex.d_res);
  TSB_CUDA(cudaGetLastError());
  h->launches += 2;
  const double tr2 = trace ? tnow() : 0;
  rc = ex.wait_result(prm.epoch, s, early);
  if (trace)
    std::fprintf(stderr, "[tsb200] first expand round: reserve+attributes %.2f ms, 2 launches %.2f ms, wait %.2f ms\n",
                 tr1 - tr0, tr2 - tr1, tnow() - tr2);
  if (rc != TSB_OK) {
    if (g_last_cuda_error.empty()) g_last_cuda_error = "expand kernels did not publish their result";
    return rc;
  }
  *n_children = ex.h_res->children;
  *n_solutions = ex.h_res->solutions;
  return TSB_OK;
}

int nq_expand(tsb_nq* h, const uint8_t* arena, const std::vector<PoolExtent>& pieces, uint8_t* children_d,
              cudaStream_t s, unsigned long long* nc, unsigned long long* ns, bool early = false) {
  return with_board(h, [&](auto n, auto r) {
    return nq_expand_n<decltype(n)::value, decltype(r)::value>(h, arena, pieces, children_d, s, nc, ns, early);
  });
}

// what a pool may hold: depth <= N, board[0..N) < N, the bytes past N zero (every node the reference or this library
// creates; the persistent kernel packs a node into 125 bits on these terms, nq_rounds_ll.cuh).  `rec`-byte records:
// {depth, board[rec - 1]}.
bool nq_nodes_valid(int N, size_t rec, const uint8_t* nodes, int64_t n) {
  for (int64_t i = 0; i < n; i++) {
    const uint8_t* x = nodes + static_cast<size_t>(i) * rec;
    if (x[0] > N) return false;
    for (size_t j = 0; j + 1 < rec; j++)
      if (x[1 + j] >= (static_cast<int>(j) < N ? N : 1)) return false;
  }
  return true;
}

template <int N, int R>
int nq_ll_launch_n(tsb_nq* h, const tsb::LlMultiParams& prm, int grid, int pools, int ppt, cudaStream_t s) {
  // (one pool: one CTA per SM; two or three: two CTAs of LL_T workers + the exchange warp per SM, capped at 112
  // registers; three or four pools: 66 CTAs per pool with 768 parents each on 132 SMs, see ll_slice.  Four pools:
  // one CTA per SM of two such halves, each running one pool (nq_rounds_ll_kernel, HALVES = 2), grid (grid, 2).
  // 25-byte records: one pool, nq_ll_grid.)
  const int halves = pools == tsb::LL_MAX_POOLS ? 2 : 1;
  void (*kernel)(const tsb::LlMultiParams);
  size_t smem;
  if constexpr (R == tsb::NQ_REC24) {
    if (pools != 1 || ppt != 2) return TSB_EINVAL;
    kernel = tsb::nq_rounds_ll_wide_kernel<N>;
    smem = sizeof(tsb::LlSmem<tsb::LL_T, 2, R>) + 128;
  } else {
    const int var = pools == 1 ? 0 : (ppt == 2 ? 1 : 2) + (halves == 2 ? 2 : 0);
    kernel = var == 0   ? tsb::nq_rounds_ll_kernel<N, tsb::LL_T, 1, 2>
             : var == 1 ? tsb::nq_rounds_ll_kernel<N, tsb::LL_T, 2, 2>
             : var == 2 ? tsb::nq_rounds_ll_kernel<N, tsb::LL_T, 2, 3>
             : var == 3 ? tsb::nq_rounds_ll_kernel<N, tsb::LL_T, 1, 2, 2>
                        : tsb::nq_rounds_ll_kernel<N, tsb::LL_T, 1, 3, 2>;
    static_assert(2 * sizeof(tsb::LlSmem<tsb::LL_T, 3>) + 128 <= 227 * 1024, "two halves' shared memory in one CTA");
    smem = halves * (ppt == 2 ? sizeof(tsb::LlSmem<tsb::LL_T, 2>) : sizeof(tsb::LlSmem<tsb::LL_T, 3>)) + 128;
  }
  int rc = h->configure(kernel, smem);
  if (rc != TSB_OK) return rc;
  void* args[] = {const_cast<tsb::LlMultiParams*>(&prm)};
  // cooperative: all CTAs of all pools co-resident (two per SM when there are two or three pools), or the launch fails
  TSB_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(kernel), dim3(grid, pools / halves),
                                       dim3(halves * (tsb::LL_T + 32)), args, smem, s));
  h->launches++;
  return TSB_OK;
}
// the plain arena's [0, pool.size) -> d_fat
template <int N, int R>
int nq_fat_import(tsb_nq* h) {
  const long long size = h->pool.size;
  if (size > 0) {
    const unsigned blocks = static_cast<unsigned>((size + 255) / 256);
    if constexpr (R == tsb::NQ_REC24)
      tsb::nq_fat_import_wide_kernel<N><<<blocks, 256, 0, h->stream>>>(h->pool.arena[h->pool.cur], h->d_fat, size);
    else
      tsb::nq_fat_import_kernel<N><<<blocks, 256, 0, h->stream>>>(h->pool.arena[h->pool.cur], h->d_fat, size);
    TSB_CUDA(cudaGetLastError());
    h->launches++;
  }
  return TSB_OK;
}
int nq_ensure_fat(tsb_nq* h, long long cap) {
  if (cap <= h->fat_cap) return TSB_OK;
  if (h->d_fat) cudaFree(h->d_fat);
  h->d_fat = nullptr;
  h->fat_cap = 0;
  TSB_CUDA(cudaMalloc(&h->d_fat, static_cast<size_t>(cap) * sizeof(tsb::FatNode)));
  h->fat_cap = cap;
  // (a new arena starts cleared: tag 0 everywhere)
  TSB_CUDA(cudaMemsetAsync(h->d_fat, 0, static_cast<size_t>(cap) * sizeof(tsb::FatNode), h->stream));
  h->tag_clear = h->rounds.epoch;
  h->tag_hi = 0;
  return TSB_OK;
}
// the clear of d_fat's tags, if the next launch (at most max_rounds rounds) needs it; -> the last epoch it may use
int nq_fat_tag_window(tsb_nq* h, int64_t max_rounds, unsigned* epoch_last, bool* queued) {
  const tsb::LlTagWindow w = tsb::ll_tag_window(h->rounds.epoch, h->tag_clear, max_rounds);
  if (w.clear) {
    const long long words = h->tag_hi * tsb::LL_WORDS;
    if (words > 0) {
      tsb::nq_fat_clear_tags_kernel<<<static_cast<unsigned>((words + 255) / 256), 256, 0, h->stream>>>(h->d_fat, words);
      TSB_CUDA(cudaGetLastError());
      h->launches++;
      *queued = true;
    }
    h->tag_clear = h->rounds.epoch;
    h->tag_hi = 0;
  }
  *epoch_last = w.epoch_last;
  return TSB_OK;
}
// the pool back in the plain arena of 21- or 25-byte records (whoever needs the node records calls this first)
int nq_materialize(tsb_nq* h) {
  if (!h->in_fat) return TSB_OK;
  TSB_CUDA(cudaSetDevice(h->device));
  const long long size = h->pool.size;
  if (size > 0) {
    auto kernel = h->wide ? tsb::nq_fat_export_wide_kernel : tsb::nq_fat_export_kernel;
    kernel<<<static_cast<unsigned>((size + 255) / 256), 256, 0, h->stream>>>(h->d_fat, h->pool.arena[h->pool.cur], size);
    TSB_CUDA(cudaGetLastError());
    h->launches++;
    TSB_CUDA(cudaStreamSynchronize(h->stream));
  }
  h->in_fat = false;
  return TSB_OK;
}
// grid (CTAs per pool) of the persistent kernel for chunks of up to M parents when one launch serves `pools` pools;
// 0: M is too large for it.  Chosen on the N = 17 search at M = 50000: one pool: 7/8 of the SMs
// (one CTA per SM); two pools: one CTA per SM each (two per SM in all); four pools: SMs / 2 CTAs each.  An all-to-all
// flag exchange among all SMs' CTAs costs 2-3x one among half of them (tools/flag_exchange.py); the per-CTA work grows
// the other way.
// *ppt: parents per thread of the kernel variant to launch (2, or 3 when the pool's CTAs would not cover M with 2).
// Wide handles (25-byte records) run one pool per launch: 0 for pools > 1.
int nq_ll_grid(const tsb_nq* h, int M, int pools, int* ppt = nullptr) {
  if (!h->di.coop || env_no_rounds() || pools < 1 || pools > (h->wide ? 1 : tsb::LL_MAX_POOLS)) return 0;
  const int sms = std::min(h->di.sms, tsb::LL_MAX_SMS);
  const int most = tsb::ll_ctas_per_pool(sms, pools);  // (ll_tiers.h: the drivers size their warm-up by the same tiers)
  const int per = static_cast<long long>(most) * tsb::ll_slice(2) >= M ? 2 : 3;
  const int slice = tsb::ll_slice(per);
  int grid = pools == 1 ? std::max(1, (sms * 7 / 8) & ~1) : most;
  while (static_cast<long long>(grid) * slice < M && grid < most) ++grid;  // (M decides)
  if (ppt) *ppt = per;
  return static_cast<long long>(M) <= static_cast<long long>(grid) * slice && (pools > 1 || per == 2) ? grid : 0;
}
// The N-Queens side of rounds_run: launches of nq_rounds_ll_kernel on the pools' fat arenas
struct NqRounds {
  using Handle = tsb_nq;
  using Sync = tsb::LlSync;
  using Params = tsb::LlMultiParams;
  static constexpr int kMaxPools = tsb::LL_MAX_POOLS;
  static constexpr const char* kKernel = "nq_rounds_ll_kernel";
  static constexpr const char* kStuck = "a flag exchange or a node poll did not complete";

  // (*ppt: the variant's parents per thread; a lone survivor gets the one-pool kernel)
  int grid(const tsb_nq* h0, int M, int pools, int* ppt) const { return nq_ll_grid(h0, M, pools, ppt); }
  int prepare(tsb_nq* h, int, int64_t left, long long need, tsb::LlParams* prm, bool* queued) const {
    DevicePool& p = h->pool;
    int rc = TSB_OK;
    if (h->in_fat && need > p.cap) rc = nq_materialize(h);  // (grows below and imports again)
    if (rc != TSB_OK) return rc;
    if (!h->in_fat) {
      // room for the worst case of the next round
      rc = p.make_stack(h->stream, need);
      if (rc == TSB_OK) rc = nq_ensure_fat(h, p.cap);
      if (rc == TSB_OK)
        rc = with_board(h, [h](auto n, auto r) { return nq_fat_import<decltype(n)::value, decltype(r)::value>(h); });
      if (rc != TSB_OK) return rc;
      h->in_fat = true;
      *queued = true;
    }
    prm->fat = h->d_fat;
    prm->cap = std::min(p.cap, h->fat_cap);
    return nq_fat_tag_window(h, left, &prm->epoch_last, queued);
  }
  int launch(tsb_nq* h0, const tsb::LlMultiParams& mp, int grid, int pools, int ppt) const {
    return with_board(h0, [&](auto n, auto r) {
      return nq_ll_launch_n<decltype(n)::value, decltype(r)::value>(h0, mp, grid, pools, ppt, h0->stream);
    });
  }
  // SPACE: back to the plain arena, which grows before the next launch; RELAUNCH (layer table full, or the tag window
  // used up): a fresh launch trusts the whole pool; DONE or PAUSE: the pool leaves
  int resume(tsb_nq* h, int, const tsb::RoundsState& st, int, int, int64_t*, uint64_t*, bool* again) const {
    h->tag_hi = std::max(h->tag_hi, st.size_hi);
    *again = st.exit_code == tsb::RND_EXIT_SPACE || st.exit_code == tsb::RND_EXIT_RELAUNCH;
    return st.exit_code == tsb::RND_EXIT_SPACE ? nq_materialize(h) : TSB_OK;
  }
  int step(tsb_nq* h, int, int m, int M, int64_t* np, uint64_t* nc, uint64_t* ns) const {
    return tsb_nq_pool_step(h, m, M, np, nc, ns);
  }
  void report(const tsb::RoundsState* pace, const int* map, int n_act, int grid) const;
  NqRounds of_pool(int) const { return *this; }
};

// TSB200_ROUNDS_PROF: CTA 0's phases of each pool, the pace of the launch and which pools shared an SM
void NqRounds::report(const tsb::RoundsState* pace, const int* map, int n_act, int grid) const {
  for (int a = 0; a < n_act; a++) {
    const tsb::RoundsState& st = pace[a];
    const double r = static_cast<double>(std::max<unsigned long long>(1, st.rounds));
    std::fprintf(stderr, "[tsb200] LL rounds kernel (pool %d of %d): %llu rounds; CTA 0 cycles per round: workers: set-up %.0f "
                 "poll-nodes %.0f scan+items %.0f build %.0f handoff-wait %.0f store %.0f | exchange warp: "
                 "scan-wait %.0f publish+plan-ahead %.0f gather-wait %.0f sums+plan %.0f handoff-wait %.0f\n", a, n_act,
                 static_cast<unsigned long long>(st.rounds), st.prof[tsb::LL_PROF_SETUP] / r, st.prof[tsb::LL_PROF_POLL] / r,
                 st.prof[tsb::LL_PROF_SCAN] / r, st.prof[tsb::LL_PROF_BUILD] / r, st.prof[tsb::LL_PROF_HAND] / r,
                 st.prof[tsb::LL_PROF_STORE] / r, st.prof[tsb::LL_PROF_X_SCAN] / r, st.prof[tsb::LL_PROF_X_AHEAD] / r,
                 st.prof[tsb::LL_PROF_X_GATHER] / r, st.prof[tsb::LL_PROF_X_TAIL] / r, st.prof[tsb::LL_PROF_X_HAND] / r);
  }
  // the pace of the launch: it ends when its last pool leaves, so a pool that leaves early idles its CTAs' SMs
  // share for the rest of it
  unsigned long long t0 = ~0ull, t1 = 0;
  for (int a = 0; a < n_act; a++) {
    t0 = std::min(t0, pace[a].t_start);
    t1 = std::max(t1, pace[a].t_exit);
  }
  for (int a = 0; a < n_act; a++) {
    const tsb::RoundsState& st = pace[a];
    const double wall = 1e-3 * static_cast<double>(st.t_exit - st.t_start);
    unsigned long long fertile = 0, wide = 0;  // (over the pool's CTAs)
    for (int c = 0; c < grid; c++) {
      fertile += st.cta_fertile[c];
      wide += st.cta_wide[c];
    }
    // why the pool left: its round budget, fewer than m nodes, a relaunch (layer table or tag window), arena room
    static const char* const why[] = {"dry", "budget", "space", "abort", "relaunch"};
    std::fprintf(stderr, "[tsb200] LL pace (pool %d of %d, handle %d): start +%.2f us, wall %.2f us, %llu rounds, "
                 "%.4f us per round, stagger %.2f us, parents %llu, children %llu, parents with children %llu, "
                 "CTA rounds over one window %llu, exit %s, globaltimer %llu..%llu ns\n", a, n_act, map[a],
                 1e-3 * static_cast<double>(st.t_start - t0), wall, static_cast<unsigned long long>(st.rounds),
                 wall / static_cast<double>(std::max<unsigned long long>(1, st.rounds)),
                 1e-3 * static_cast<double>(t1 - st.t_exit), static_cast<unsigned long long>(st.parents),
                 static_cast<unsigned long long>(st.children), fertile, wide,
                 st.exit_code >= 0 && st.exit_code <= tsb::RND_EXIT_RELAUNCH ? why[st.exit_code] : "?", st.t_start,
                 st.t_exit);
  }
  // residency: which pools' CTAs share an SM, and which of them started there first
  int row_of[2][tsb::LL_MAX_SMS * 2], n_on[tsb::LL_MAX_SMS * 2] = {};
  unsigned t_of[2][tsb::LL_MAX_SMS * 2];
  for (int a = 0; a < n_act; a++)
    for (int c = 0; c < grid; c++) {
      const unsigned s = pace[a].cta_sm[c] % (tsb::LL_MAX_SMS * 2);
      if (n_on[s] < 2) {
        row_of[n_on[s]][s] = a;
        t_of[n_on[s]][s] = pace[a].cta_t0[c];
      }
      n_on[s]++;
    }
  int pairs[tsb::LL_MAX_POOLS][tsb::LL_MAX_POOLS] = {}, first[tsb::LL_MAX_POOLS] = {}, over = 0;
  for (int s = 0; s < tsb::LL_MAX_SMS * 2; s++) {
    if (n_on[s] > 2) over++;
    if (n_on[s] < 2) continue;
    const bool zero_first = static_cast<int>(t_of[1][s] - t_of[0][s]) >= 0;
    const int lo = std::min(row_of[0][s], row_of[1][s]), hi = std::max(row_of[0][s], row_of[1][s]);
    pairs[lo][hi]++;
    first[zero_first ? row_of[0][s] : row_of[1][s]]++;
  }
  std::string sh;
  for (int x = 0; x < n_act; x++)
    for (int y = x; y < n_act; y++)
      if (pairs[x][y]) sh += " " + std::to_string(x) + "+" + std::to_string(y) + ": " + std::to_string(pairs[x][y]);
  std::string fs;
  for (int x = 0; x < n_act; x++) fs += " " + std::to_string(x) + ": " + std::to_string(first[x]);
  std::fprintf(stderr, "[tsb200] LL residency: SMs shared by pools%s | started first on a shared SM, by pool%s | SMs "
               "with more than two CTAs: %d\n", sh.c_str(), fs.c_str(), over);
}

// ============================================================================ PFSP
template <int KIND, int M, bool SIMD>
int launch_lb1_km(tsb_pfsp* h, const uint8_t* in, uint8_t* out, long long count, cudaStream_t s) {
  auto kernel = tsb::pfsp_lb1_kernel<KIND, M, SIMD>;
  const size_t smem = sizeof(tsb::Lb1Smem) + 128;
  int grid = 1;
  int rc = h->grid_for(kernel, tsb::PF_THREADS, smem, count, tsb::PF_TILE, &grid);
  if (rc != TSB_OK) return rc;
  kernel<<<grid, tsb::PF_THREADS, smem, s>>>(in, out, count, h->d_tab1);
  TSB_CUDA(cudaGetLastError());
  h->launches++;
  return TSB_OK;
}

template <int M, typename CT>
int launch_lb2_mc(tsb_pfsp* h, const CT& C, const uint8_t* in, uint8_t* out, long long count, int best, cudaStream_t s) {
  auto kernel = tsb::pfsp_lb2_kernel<M, CT>;
  const size_t smem = sizeof(tsb::Lb2Smem<M>) + 128;
  int grid = 1;
  int rc = h->grid_for(kernel, tsb::PF_THREADS, smem, count, tsb::LB2_TILE, &grid);
  if (rc != TSB_OK) return rc;
  kernel<<<grid, tsb::PF_THREADS, smem, s>>>(in, out, count, h->d_tab1, C, best);
  TSB_CUDA(cudaGetLastError());
  h->launches++;
  return TSB_OK;
}
template <int M>
int launch_lb2_m(tsb_pfsp* h, const uint8_t* in, uint8_t* out, long long count, int best, cudaStream_t s) {
  if constexpr (M <= 10) {
    if (h->d_tabu) return launch_lb2_mc<M>(h, tsb::Lb2ConstU{h->d_tabu}, in, out, count, best, s);
  }
  return launch_lb2_mc<M>(h, h->tab->lb2c, in, out, count, best, s);
}

template <int KIND, int M>
int launch_wide_km(tsb_pfsp* h, const uint8_t* in, uint8_t* out, long long count, int best, cudaStream_t s) {
  auto kernel = tsb::pfsp_wide_kernel<KIND, M>;
  const size_t smem = sizeof(tsb::PfspWideSmem) + 128;
  int grid = 1;
  int rc = h->grid_for(kernel, tsb::PW_THREADS, smem, count + tsb::PW_TILE - 1, tsb::PW_TILE, &grid);
  if (rc != TSB_OK) return rc;
  kernel<<<grid, tsb::PW_THREADS, smem, s>>>(in, reinterpret_cast<int32_t*>(out), count, h->d_wtab, best);
  TSB_CUDA(cudaGetLastError());
  h->launches++;
  return TSB_OK;
}
template <int M>
int launch_wide_m(tsb_pfsp* h, int lb_kind, const uint8_t* in, uint8_t* out, long long count, int best, cudaStream_t s) {
  if (lb_kind == TSB_LB1_D) return launch_wide_km<0, M>(h, in, out, count, best, s);
  if (lb_kind == TSB_LB1) return launch_wide_km<1, M>(h, in, out, count, best, s);
  return launch_wide_km<2, M>(h, in, out, count, best, s);
}

int launch_pfsp(tsb_pfsp* h, int lb_kind, const uint8_t* in, uint8_t* out, long long count, int64_t best64,
                cudaStream_t s) {
  const int best = clamp_best(best64);
  return with_machines(h->tab->mt, [&](auto mt) {
    constexpr int M = decltype(mt)::value;
    if (h->tab->wide) return launch_wide_m<M>(h, lb_kind, in, out, count, best, s);
    if (lb_kind == TSB_LB1)
      return h->tab->simd16 ? launch_lb1_km<1, M, true>(h, in, out, count, s) : launch_lb1_km<1, M, false>(h, in, out, count, s);
    if (lb_kind == TSB_LB1_D)
      return h->tab->simd16 ? launch_lb1_km<0, M, true>(h, in, out, count, s) : launch_lb1_km<0, M, false>(h, in, out, count, s);
    return launch_lb2_m<M>(h, in, out, count, best, s);
  });
}

template <int M>
int pfsp_expand_m(tsb_pfsp* h, int lb_kind, const uint8_t* arena, const tsb::ExpandParams& prm, uint8_t* children_d,
                  cudaStream_t s) {
  ExpandCtx& ex = h->ex;
  const long long recs = static_cast<long long>(prm.n_tiles) * tsb::PF_TILE;
  auto k3 = tsb::pfsp_expand_build_kernel;
  const size_t smem3 = sizeof(tsb::PfBuildSmem) + 128;
  int g1 = 1, g3 = 1;
  int rc = h->grid_for(k3, tsb::PF_THREADS, smem3, recs, tsb::PF_TILE, &g3);
  if (rc != TSB_OK) return rc;
  if ((prm.n_tiles + g3 - 1) / g3 > tsb::EXP_MAX_OWN) return TSB_EINVAL;
  if (lb_kind == TSB_LB2) {
    const size_t smem1 = sizeof(tsb::Lb2CountSmem<M>) + 128;
    // (this kernel walks the round in half tiles and accumulates the tile counts)
    TSB_CUDA(cudaMemsetAsync(ex.d_tile, 0, static_cast<size_t>(prm.n_tiles) * sizeof(int), s));
    auto go = [&](auto k1, const auto& C) -> int {
      int r2 = h->grid_for(k1, tsb::PF_THREADS, smem1, recs, tsb::LB2_TILE, &g1);
      if (r2 != TSB_OK) return r2;
      k1<<<g1, tsb::PF_THREADS, smem1, s>>>(arena, prm, h->d_tab1, C, ex.d_cmask, ex.d_tile, ex.d_st);
      return TSB_OK;
    };
    bool done = false;
    if constexpr (M <= 10) {
      if (h->d_tabu) {
        rc = go(tsb::pfsp_expand_count_lb2_kernel<M, tsb::Lb2ConstU>, tsb::Lb2ConstU{h->d_tabu});
        done = true;
      }
    }
    if (!done) rc = go(tsb::pfsp_expand_count_lb2_kernel<M, tsb::Lb2Const>, h->tab->lb2c);
    if (rc != TSB_OK) return rc;
  } else {
    auto k1 = lb_kind == TSB_LB1
                  ? (h->tab->simd16 ? tsb::pfsp_expand_count_lb1_kernel<1, M, true> : tsb::pfsp_expand_count_lb1_kernel<1, M, false>)
                  : (h->tab->simd16 ? tsb::pfsp_expand_count_lb1_kernel<0, M, true> : tsb::pfsp_expand_count_lb1_kernel<0, M, false>);
    const size_t smem1 = sizeof(tsb::Lb1CountSmem) + 128;
    rc = h->grid_for(k1, tsb::PF_THREADS, smem1, recs, tsb::PF_TILE, &g1);
    if (rc != TSB_OK) return rc;
    k1<<<g1, tsb::PF_THREADS, smem1, s>>>(arena, prm, h->d_tab1, ex.d_cmask, ex.d_tile, ex.d_st);
  }
  k3<<<g3, tsb::PF_THREADS, smem3, s>>>(arena, prm, ex.d_cmask, ex.d_tile, children_d, ex.d_st, ex.d_res);
  TSB_CUDA(cudaGetLastError());
  h->launches += 2;
  return TSB_OK;
}

// the same round on a 50-job handle (pfsp_wide_expand.cuh): count, build
template <int M>
int pfsp_wide_expand_m(tsb_pfsp* h, int lb_kind, const uint8_t* arena, const tsb::ExpandParams& prm,
                       uint8_t* children_d, cudaStream_t s) {
  ExpandCtx& ex = h->ex;
  const long long recs = static_cast<long long>(prm.n_tiles) * tsb::PW_TILE;
  auto k1 = lb_kind == TSB_LB1_D ? tsb::pfsp_wide_expand_count_kernel<0, M>
            : lb_kind == TSB_LB1 ? tsb::pfsp_wide_expand_count_kernel<1, M>
                                 : tsb::pfsp_wide_expand_count_kernel<2, M>;
  auto k3 = tsb::pfsp_wide_expand_build_kernel;
  const size_t smem1 = sizeof(tsb::PfspWideCountSmem) + 128, smem3 = sizeof(tsb::PfspWideBuildSmem) + 128;
  int g1 = 1, g3 = 1;
  int rc = h->grid_for(k1, tsb::PW_THREADS, smem1, recs, tsb::PW_TILE, &g1);
  if (rc == TSB_OK) rc = h->grid_for(k3, tsb::PW_THREADS, smem3, recs, tsb::PW_TILE, &g3);
  if (rc != TSB_OK) return rc;
  if ((prm.n_tiles + g3 - 1) / g3 > tsb::EXP_MAX_OWN) return TSB_EINVAL;
  auto* d_mask = reinterpret_cast<unsigned long long*>(ex.d_cmask);
  k1<<<g1, tsb::PW_THREADS, smem1, s>>>(arena, prm, h->d_wtab, d_mask, ex.d_tile, ex.d_st);
  k3<<<g3, tsb::PW_THREADS, smem3, s>>>(arena, prm, d_mask, ex.d_tile, children_d, ex.d_st, ex.d_res);
  TSB_CUDA(cudaGetLastError());
  h->launches += 2;
  return TSB_OK;
}

// generate_children of pfsp_gpu_chpl.chpl:273-303 on host arrays (the sequential rule, used by the slow path)
template <class Node>
void pfsp_generate_children_host(int jobs, const Node* parents, int size, const int32_t* bounds, int64_t* best,
                                 std::vector<Node>* kids, uint64_t* sol) {
  for (int i = 0; i < size; i++) {
    const Node& parent = parents[i];
    const int depth = parent.depth;
    for (int j = parent.limit1 + 1; j < jobs; j++) {
      const int32_t lb = bounds[j + static_cast<size_t>(i) * jobs];
      if (depth + 1 == jobs) {
        ++*sol;
        if (lb < *best) *best = lb;
      } else if (lb < *best) {
        Node c = parent;
        c.depth = depth + 1;
        c.limit1 = parent.limit1 + 1;
        std::swap(c.prmu[depth], c.prmu[j]);
        kids->push_back(c);
      }
    }
  }
}

// One evaluate + generate_children round over `pieces` of `arena`; children packed at `children_d` (room for
// n * jobs nodes).  *best is read and updated with the reference's semantics.  Synchronous.
int pfsp_expand_round(tsb_pfsp* h, int lb_kind, const uint8_t* arena, const std::vector<PoolExtent>& pieces,
                      uint8_t* children_d, cudaStream_t s, int64_t* best, unsigned long long* n_children,
                      unsigned long long* n_solutions, bool early = false) {
  tsb::ExpandParams prm;
  const bool wide = h->tab->wide;
  const int tile = wide ? tsb::PW_TILE : tsb::PF_TILE;
  int rc = make_params(pieces, tile, &prm);
  if (rc != TSB_OK) return rc;
  const int best_launch = clamp_best(*best);
  ExpandCtx& ex = h->ex;
  // (side array: one child mask per parent, 32 bits for 20 jobs, 64 for 50)
  rc = ex.reserve(std::max<long long>(prm.n_tiles, h->M_max / tile + 2 * tsb::EXP_MAX_PIECES), wide ? tile * 8 : tile * 4, s);
  if (rc != TSB_OK) return rc;
  prm.epoch = ++ex.epoch;
  prm.best = best_launch;
  rc = with_machines(h->tab->mt, [&](auto mt) {
    constexpr int M = decltype(mt)::value;
    return wide ? pfsp_wide_expand_m<M>(h, lb_kind, arena, prm, children_d, s)
                : pfsp_expand_m<M>(h, lb_kind, arena, prm, children_d, s);
  });
  if (rc != TSB_OK) return rc;
  rc = ex.wait_result(prm.epoch, s, early);
  if (rc != TSB_OK) {
    if (g_last_cuda_error.empty()) g_last_cuda_error = "expand kernels did not publish their result";
    return rc;
  }
  if (ex.h_res->best >= best_launch) {  // no leaf of the chunk improved best: the launch-value masks are exact
    *n_children = ex.h_res->children;
    *n_solutions = ex.h_res->solutions;
    return TSB_OK;
  }
  // ---- slow path: a leaf lowered best inside this chunk, which changes what the rest of the chunk pushes
  // (sequential rule).  Redo the round: bounds through the evaluator, children on the host.
  ++h->slow_rounds;
  long long n = 0;
  for (const PoolExtent& x : pieces) n += x.e - x.b;
  if (n > h->M_max) return TSB_EINVAL;  // (cannot happen: every entry point checks count <= M_max first)
  const size_t rec = h->in_rec;  // (the node record: 88 or 208 bytes)
  long long at = 0;
  if (!(arena == h->d_in && pieces.size() == 1 && pieces[0].b == 0))
    for (const PoolExtent& x : pieces) {  // the chunk, contiguous
      TSB_CUDA(cudaMemcpyAsync(h->d_in + at * rec, arena + x.b * rec, static_cast<size_t>(x.e - x.b) * rec,
                               cudaMemcpyDeviceToDevice, s));
      at += x.e - x.b;
    }
  rc = launch_pfsp(h, lb_kind, h->d_in, h->d_out, n, *best, s);
  if (rc != TSB_OK) return rc;
  const auto redo = [&](auto& chunk, auto& kids) -> int {
    using Node = typename std::decay_t<decltype(chunk)>::value_type;
    chunk.resize(static_cast<size_t>(n));
    h->h_bounds.resize(static_cast<size_t>(n) * h->tab->jobs);
    int r = h->copy_d2h(chunk.data(), h->d_in, static_cast<size_t>(n) * sizeof(Node), s);
    if (r == TSB_OK) r = h->copy_d2h(h->h_bounds.data(), h->d_out, static_cast<size_t>(n) * h->tab->jobs * 4, s);
    if (r != TSB_OK) return r;
    kids.clear();
    uint64_t sol = 0;
    pfsp_generate_children_host(h->tab->jobs, chunk.data(), static_cast<int>(n), h->h_bounds.data(), best, &kids, &sol);
    r = h->copy_h2d(children_d, kids.data(), kids.size() * sizeof(Node), s);
    if (r != TSB_OK) return r;
    *n_children = kids.size();
    *n_solutions = sol;
    return TSB_OK;
  };
  return wide ? redo(h->h_chunk50, h->h_kids50) : redo(h->h_chunk, h->h_kids);
}

// (the PFSP pool only ever lives in its plain arena)
int pfsp_plain() { return TSB_OK; }

// one round of h's device pool (tsb_pfsp_pool_step after its checks; on 50-job handles, the searches' rounds)
int pfsp_step(tsb_pfsp* h, int lb_kind, int m, int M, int64_t* best, int64_t* n_parents, uint64_t* n_children,
              uint64_t* n_solutions) {
  return pool_step(*h, m, M, n_parents, n_children, n_solutions, pfsp_plain,
                   [h, lb_kind, best](auto arena, const auto& pieces, auto kids, auto nc, auto ns) {
                     return pfsp_expand_round(h, lb_kind, arena, pieces, kids, h->stream, best, nc, ns, /*early=*/true);
                   });
}

// CTAs of the persistent PFSP kernel for chunks of up to M parents (one per SM at most, each with up to PFR_SLICE
// parents; fewer CTAs for smaller M, so that the two exchanges of a round involve only the CTAs that have parents to
// evaluate); 0: the loop of tsb_pfsp_pool_step runs instead (lb2, M above PFR_MAX_M where the step loop is faster, M
// beyond pf_pool_capacity, no cooperative launch, env TSB200_NO_ROUNDS=1, a 50-job handle)
int pfsp_rounds_grid(const tsb_pfsp* h, int lb_kind, int M) {
  if (lb_kind == TSB_LB2 || h->tab->wide || !h->di.coop || env_no_rounds()) return 0;
  if (M > tsb::PFR_MAX_M || M > tsb::pf_pool_capacity(h->di.sms, 1)) return 0;
  return static_cast<int>(std::min<long long>(tsb::pf_ctas_per_pool(h->di.sms, 1),
                                              (static_cast<long long>(M) + tsb::PF_TILE - 1) / tsb::PF_TILE));
}
// f(kernel): the persistent kernel of h's route for lb1 / lb1_d
template <class F>
int with_pfsp_rounds_kernel(const tsb_pfsp* h, int lb_kind, F&& f) {
  return with_machines(h->tab->mt, [&](auto mt) -> int {
    constexpr int MT = decltype(mt)::value;
    if (lb_kind == TSB_LB1) return h->tab->simd16 ? f(tsb::pfsp_rounds_kernel<1, MT, true>) : f(tsb::pfsp_rounds_kernel<1, MT, false>);
    return h->tab->simd16 ? f(tsb::pfsp_rounds_kernel<0, MT, true>) : f(tsb::pfsp_rounds_kernel<0, MT, false>);
  });
}
constexpr size_t kPfRoundsSmem = sizeof(tsb::PfRoundsSmem) + 128;
// CTAs per pool when one launch of the persistent kernel serves `pools` >= 2 pools with chunks of up to M parents
// (pf_ctas_per_pool, fewer for small M as in pfsp_rounds_grid); 0: not in one launch (lb2, no cooperative launch, env
// TSB200_NO_ROUNDS=1, a 50-job handle, M beyond pf_pool_capacity, or the kernel does not fit twice on an SM)
int pfsp_multi_grid(tsb_pfsp* h, int lb_kind, int M, int pools) {
  if (lb_kind == TSB_LB2 || h->tab->wide || !h->di.coop || env_no_rounds() || pools < 2 || pools > tsb::PFR_MAX_POOLS) return 0;
  if (M > tsb::pf_pool_capacity(h->di.sms, pools)) return 0;
  int per_sm = 0;
  if (with_pfsp_rounds_kernel(h, lb_kind, [&](auto kernel) -> int {
        return h->per_sm(kernel, tsb::PF_THREADS, kPfRoundsSmem, &per_sm);
      }) != TSB_OK || per_sm < 2) {
    (void)cudaGetLastError();
    return 0;
  }
  return static_cast<int>(std::min<long long>(tsb::pf_ctas_per_pool(h->di.sms, pools),
                                              (static_cast<long long>(M) + tsb::PF_TILE - 1) / tsb::PF_TILE));
}
int pfsp_rounds_launch(tsb_pfsp* h, int lb_kind, const tsb::PfRoundsMultiParams& prm, int grid, int pools, cudaStream_t s) {
  return with_pfsp_rounds_kernel(h, lb_kind, [&](auto kernel) -> int {
    int rc = h->configure(kernel, kPfRoundsSmem);
    if (rc != TSB_OK) return rc;
    void* args[] = {const_cast<tsb::PfRoundsMultiParams*>(&prm)};
    // cooperative: every CTA of every pool co-resident (the exchanges wait for all of a pool's CTAs), or the launch fails
    TSB_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(kernel), dim3(grid, pools), dim3(tsb::PF_THREADS), args,
                                         kPfRoundsSmem, s));
    h->launches++;
    return TSB_OK;
  });
}
// The PFSP side of rounds_run: launches of pfsp_rounds_kernel on the pools' plain arenas; best[i] is pool i's
// incumbent
struct PfspRounds {
  using Handle = tsb_pfsp;
  using Sync = tsb::PfRoundsSync;
  using Params = tsb::PfRoundsMultiParams;
  static constexpr int kMaxPools = tsb::PFR_MAX_POOLS;
  static constexpr const char* kKernel = "pfsp_rounds_kernel";
  static constexpr const char* kStuck = "a count or store exchange did not complete";
  int lb_kind;
  int64_t* best;

  int grid(tsb_pfsp* h0, int M, int pools, int*) const {
    return pools == 1 ? pfsp_rounds_grid(h0, lb_kind, M) : pfsp_multi_grid(h0, lb_kind, M, pools);
  }
  int prepare(tsb_pfsp* h, int i, int64_t, long long need, tsb::PfRoundsParams* prm, bool* queued) const {
    DevicePool& p = h->pool;
    const int rc = p.make_stack(h->stream, need);  // room for the worst case of the next round
    prm->arena = p.arena[p.cur];
    prm->tables = h->d_tab1;
    prm->cap = p.cap;
    prm->best = clamp_best(best[i]);
    *queued = true;  // (a pool_step round may still be storing on h's stream)
    return rc;
  }
  int launch(tsb_pfsp* h0, const tsb::PfRoundsMultiParams& mp, int grid, int pools, int) const {
    return pfsp_rounds_launch(h0, lb_kind, mp, grid, pools, h0->stream);
  }
  // SPACE: the arena grows before the next launch; IMPROVED: a leaf of the chunk improved best[i], so that round goes
  // through tsb_pfsp_pool_step and its sequential rule and the pool goes again with the new incumbent; DONE or PAUSE:
  // the pool leaves
  int resume(tsb_pfsp* h, int i, const tsb::RoundsState& st, int m, int M, int64_t* left, uint64_t* out, bool* again) const {
    *again = st.exit_code == tsb::RND_EXIT_SPACE || st.exit_code == tsb::PFR_EXIT_IMPROVED;
    if (st.exit_code != tsb::PFR_EXIT_IMPROVED) return TSB_OK;
    --*left;
    return step_loop(1, out, [&](int64_t* np, uint64_t* nc, uint64_t* ns) { return step(h, i, m, M, np, nc, ns); });
  }
  int step(tsb_pfsp* h, int i, int m, int M, int64_t* np, uint64_t* nc, uint64_t* ns) const {
    return pfsp_step(h, lb_kind, m, M, &best[i], np, nc, ns);
  }
  // TSB200_ROUNDS_PROF: CTA 0's phases of each pool
  void report(const tsb::RoundsState* pace, const int*, int n_act, int) const {
    for (int a = 0; a < n_act; a++) {
      const tsb::RoundsState& st = pace[a];
      const double r = static_cast<double>(std::max<unsigned long long>(1, st.rounds));
      std::fprintf(stderr, "[tsb200] PFSP rounds kernel (pool %d of %d): %llu rounds (exit %d); CTA 0 cycles per round: "
                   "load %.0f bounds %.0f publish+items %.0f gather %.0f store %.0f store-exchange %.0f\n", a, n_act,
                   static_cast<unsigned long long>(st.rounds), st.exit_code, st.prof[tsb::PFR_PROF_LOAD] / r,
                   st.prof[tsb::PFR_PROF_BOUND] / r, st.prof[tsb::PFR_PROF_PUBLISH] / r, st.prof[tsb::PFR_PROF_GATHER] / r,
                   st.prof[tsb::PFR_PROF_STORE] / r, st.prof[tsb::PFR_PROF_BARRIER] / r);
    }
  }
  PfspRounds of_pool(int i) const { return {lb_kind, best + i}; }
};

// ---- the same for 50-job handles: pfsp_wide_rounds_kernel (pfsp_wide_rounds.cuh) on 208-byte records
constexpr size_t kPfWideRoundsSmem = sizeof(tsb::PfWideRoundsSmem) + 128;
template <class F>
int with_pfsp_wide_rounds_kernel(const tsb_pfsp* h, int lb_kind, F&& f) {
  return with_machines(h->tab->mt, [&](auto mt) -> int {
    constexpr int MT = decltype(mt)::value;
    return lb_kind == TSB_LB1 ? f(tsb::pfsp_wide_rounds_kernel<1, MT>) : f(tsb::pfsp_wide_rounds_kernel<0, MT>);
  });
}
// CTAs per pool of a launch that serves `pools` 50-job pools with chunks of up to M parents (pf_ctas_per_pool, fewer
// for small M, as in pfsp_rounds_grid); 0: the pools run the step loop of pfsp_step instead (lb2, no cooperative
// launch, env TSB200_NO_ROUNDS=1, M beyond pfw_takes, or, for several pools, the kernel does not fit twice on an SM)
int pfsp_wide_grid(tsb_pfsp* h, int lb_kind, int M, int pools) {
  if (lb_kind == TSB_LB2 || !h->di.coop || env_no_rounds() || !tsb::pfw_takes(h->di.sms, pools, M)) return 0;
  int per_sm = 0;
  if (with_pfsp_wide_rounds_kernel(h, lb_kind, [&](auto kernel) -> int {
        return h->per_sm(kernel, tsb::PFW_THREADS, kPfWideRoundsSmem, &per_sm);
      }) != TSB_OK || per_sm < (pools == 1 ? 1 : 2)) {
    (void)cudaGetLastError();
    return 0;
  }
  return static_cast<int>(std::min<long long>(tsb::pf_ctas_per_pool(h->di.sms, pools),
                                              (static_cast<long long>(M) + tsb::PFW_TILE - 1) / tsb::PFW_TILE));
}
// The 50-job side of rounds_run: PfspRounds with the wide kernel, tables and launch shape
struct PfspWideRounds : PfspRounds {
  using Params = tsb::PfWideRoundsMultiParams;
  static constexpr const char* kKernel = "pfsp_wide_rounds_kernel";

  int grid(tsb_pfsp* h0, int M, int pools, int*) const { return pfsp_wide_grid(h0, lb_kind, M, pools); }
  int prepare(tsb_pfsp* h, int i, int64_t, long long need, tsb::PfWideRoundsParams* prm, bool* queued) const {
    DevicePool& p = h->pool;
    const int rc = p.make_stack(h->stream, need);  // room for the worst case of the next round
    prm->arena = p.arena[p.cur];
    prm->tables = h->d_wtab;
    prm->cap = p.cap;
    prm->best = clamp_best(best[i]);
    *queued = true;  // (a pfsp_step round may still be storing on h's stream)
    return rc;
  }
  int launch(tsb_pfsp* h0, const tsb::PfWideRoundsMultiParams& mp, int grid, int pools, int) const {
    return with_pfsp_wide_rounds_kernel(h0, lb_kind, [&](auto kernel) -> int {
      int rc = h0->configure(kernel, kPfWideRoundsSmem);
      if (rc != TSB_OK) return rc;
      void* args[] = {const_cast<tsb::PfWideRoundsMultiParams*>(&mp)};
      // cooperative: every CTA of every pool co-resident (the exchanges wait for all of a pool's CTAs), or the launch fails
      TSB_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(kernel), dim3(grid, pools), dim3(tsb::PFW_THREADS),
                                           args, kPfWideRoundsSmem, h0->stream));
      h0->launches++;
      return TSB_OK;
    });
  }
  // TSB200_ROUNDS_PROF: CTA 0's phases of each pool
  void report(const tsb::RoundsState* pace, const int*, int n_act, int grid) const {
    for (int a = 0; a < n_act; a++) {
      const tsb::RoundsState& st = pace[a];
      const double r = static_cast<double>(std::max<unsigned long long>(1, st.rounds));
      std::fprintf(stderr, "[tsb200] PFSP 50-job rounds kernel (pool %d of %d, %d CTAs): %llu rounds (exit %d); CTA 0 "
                   "cycles per round: load %.0f bounds %.0f publish %.0f gather %.0f store %.0f store-exchange %.0f\n",
                   a, n_act, grid, static_cast<unsigned long long>(st.rounds), st.exit_code,
                   st.prof[tsb::PFR_PROF_LOAD] / r, st.prof[tsb::PFR_PROF_BOUND] / r, st.prof[tsb::PFR_PROF_PUBLISH] / r,
                   st.prof[tsb::PFR_PROF_GATHER] / r, st.prof[tsb::PFR_PROF_STORE] / r, st.prof[tsb::PFR_PROF_BARRIER] / r);
    }
  }
  PfspWideRounds of_pool(int i) const { return {{lb_kind, best + i}}; }
};

// A handle with chunks of up to M_max parents on `device`, an empty pool and the tables `tab` (its own, or its owner's
// for a sibling).  Tables with an index out of range give TSB_EINVAL, after the errors of the device itself.
int pfsp_open(int device, int M_max, std::shared_ptr<const PfspPacked> tab, tsb_pfsp** out) {
  tsb_pfsp* h = new (std::nothrow) tsb_pfsp();
  if (!h) return TSB_ENOMEM;
  h->tab = std::move(tab);
  const PfspPacked& t = *h->tab;
  const size_t rec = t.wide ? tsb::PW_REC : sizeof(tsb_pfsp_node);
  if (t.wide)
    // (208-byte nodes start on a 16-byte boundary anywhere.)  The arena starts with room for one worst-case round
    // (every slot of M_max parents survives) above a pool of 2 M_max nodes: 2.6 M nodes, 541 MB at M = 50000.  The
    // 20-job rule (four worst-case rounds) would be 2 GB per arena, and a search task holds two arenas per pool,
    // pools per task and tasks per GPU; a 50-job search under --ub 1 keeps far fewer nodes than its worst case, and
    // a pool that does outgrow the arena doubles it (DevicePool::reserve).
    h->pool.set_format(rec, tsb::PW_TILE, 1, t.jobs, std::max<long long>(1LL << 16, static_cast<long long>(M_max) * (t.jobs + 2)));
  else  // (88-byte nodes: extents on even records start on a 16-byte boundary)
    h->pool.set_format(rec, tsb::PF_TILE, 2, t.jobs, std::max<long long>(1LL << 20, 4LL * M_max * t.jobs));
  int rc = h->init(device, M_max, rec, static_cast<size_t>(t.jobs) * 4);
  if (rc == TSB_OK && !t.valid) rc = TSB_EINVAL;
  auto upload = [h](auto** dst, const auto& src) -> int {
    TSB_CUDA(cudaMalloc(dst, sizeof(src)));
    TSB_CUDA(cudaMemcpyAsync(*dst, &src, sizeof(src), cudaMemcpyHostToDevice, h->stream));
    TSB_CUDA(cudaStreamSynchronize(h->stream));
    return TSB_OK;
  };
  if (rc == TSB_OK) rc = t.wide ? upload(&h->d_wtab, t.tw) : upload(&h->d_tab1, t.t1);
  if (rc == TSB_OK && t.lb2u) rc = upload(&h->d_tabu, t.tabu);
  if (rc != TSB_OK) {
    destroy(h);
    return rc;
  }
  *out = h;
  return TSB_OK;
}

// The checks of a PFSP entry point on its handle and bound: TSB_EINVAL for a null handle, an unknown bound or lb2 on
// a handle without machine pairs.  `pool`: an entry point of the fused expand or the device pool, which exist for
// 20 jobs only: TSB_EUNSUPPORTED first on a 50-job handle.
int pfsp_check(const tsb_pfsp* h, bool pool, int lb_kind = TSB_LB1) {
  if (!h) return TSB_EINVAL;
  if (pool && h->tab->wide) return TSB_EUNSUPPORTED;
  if (lb_kind < 0 || lb_kind > 2 || (lb_kind == TSB_LB2 && h->tab->pairs == 0)) return TSB_EINVAL;
  return TSB_OK;
}

}  // namespace

// ============================================================================ exported C ABI
extern "C" {

const char* tsb_version(void) { return "tsb200 0.1 (sm_90a)"; }

int tsb_device_sm_count(int device) {
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  return n;
}

const char* tsb_strerror(int code) {
  switch (code) {
    case TSB_OK: return "ok";
    case TSB_EINVAL: return "invalid argument";
    case TSB_ECUDA: return "CUDA runtime error (see tsb_last_cuda_error)";
    case TSB_ENOMEM: return "out of memory";
    case TSB_ENODEV: return "no such CUDA device";
    case TSB_EALIGN: return "device pointer not 16-byte aligned";
    case TSB_EUNSUPPORTED: return "unsupported instance shape (jobs must be 20, machines 1..20)";
    case TSB_ESTOPPED: return "search stopped; its checkpoint file holds it";
  }
  return "unknown error";
}
const char* tsb_last_cuda_error(void) { return g_last_cuda_error.c_str(); }

int tsb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    (void)cudaGetLastError();
    return TSB_ENODEV;
  }
  return n;
}

// NUMA placement of a host thread that feeds one GPU (SCALE_r01: eight zero-copy streams through one socket's
// memory controllers and the inter-socket link cost half of the 8-GPU e2e throughput): pin the CALLING thread to
// the cores local to `device` (sysfs local_cpulist of its PCI function); pages the thread touches first afterwards
// — its chunk arrays, the library's pinned staging buffers — then live on that GPU's NUMA node.
int tsb_bind_thread_to_device(int device) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) {
    (void)cudaGetLastError();
    return TSB_ENODEV;
  }
  char bus[64] = {0};
  TSB_CUDA(cudaDeviceGetPCIBusId(bus, sizeof(bus) - 1, device));
  for (char* c = bus; *c; ++c) *c = static_cast<char>(std::tolower(static_cast<unsigned char>(*c)));
  const std::string path = std::string("/sys/bus/pci/devices/") + bus + "/local_cpulist";
  std::FILE* f = std::fopen(path.c_str(), "r");
  if (!f) return TSB_EUNSUPPORTED;
  char line[4096] = {0};
  const bool got = std::fgets(line, sizeof(line) - 1, f) != nullptr;
  std::fclose(f);
  if (!got) return TSB_EUNSUPPORTED;
  cpu_set_t want, have;
  CPU_ZERO(&want);
  int count = 0;
  for (const char* p = line; *p;) {  // "0-31,64-95"
    char* end = nullptr;
    const long a = std::strtol(p, &end, 10);
    if (end == p) break;
    long b = a;
    p = end;
    if (*p == '-') {
      b = std::strtol(p + 1, &end, 10);
      p = end;
    }
    for (long c = a; c <= b && c < CPU_SETSIZE; c++) CPU_SET(static_cast<int>(c), &want);
    if (*p == ',') ++p;
  }
  if (sched_getaffinity(0, sizeof(have), &have) != 0) return TSB_EUNSUPPORTED;
  cpu_set_t both;
  CPU_AND(&both, &want, &have);  // never outside what the process was given (containers, taskset)
  count = CPU_COUNT(&both);
  if (count == 0) return TSB_EUNSUPPORTED;
  if (sched_setaffinity(0, sizeof(both), &both) != 0) return TSB_EUNSUPPORTED;
  return count;
}

int tsb_init_devices(int n) {
  int have = 0;
  if (cudaGetDeviceCount(&have) != cudaSuccess || have < 1) {
    (void)cudaGetLastError();
    return TSB_ENODEV;
  }
  for (int d = 0; d < n && d < have; d++) {
    TSB_CUDA(cudaSetDevice(d));
    TSB_CUDA(cudaFree(nullptr));
    // the library's kernels are loaded lazily, as one module, at the first launch (~15 ms): do it here, where
    // the Chapel runtime loads its own GPU code — at program start, outside the drivers' timers
    cudaFuncAttributes fa;
    TSB_CUDA(cudaFuncGetAttributes(&fa, tsb::nq_evaluate_kernel<1>));
  }
  // peer access between the devices of a multi-GPU search, once and before any timer (the first
  // cudaDeviceEnablePeerAccess of a pair takes milliseconds): steals between device pools then go GPU to GPU
  // peer-to-peer instead of being staged through the host
  static std::mutex peer_mu;
  static bool peer_on[16][16] = {};
  std::lock_guard<std::mutex> lk(peer_mu);
  const int nd = std::min(std::min(n, have), 16);
  for (int a = 0; a < nd && nd > 1; a++)
    for (int b = 0; b < nd; b++)
      if (a != b && !peer_on[a][b]) {
        enable_peer(a, b);
        peer_on[a][b] = true;
      }
  return TSB_OK;
}

// diagnostics: cycles per round of bare flag exchanges among co-resident CTAs (rounds_sync_bench_kernel, nq_rounds_ll.cuh)
int tsb_debug_flag_exchange(int device, int rounds, int variant, int ctas, double* cycles_per_round) {
  if (!cycles_per_round || rounds < 1) return TSB_EINVAL;
  DeviceInfo di;
  int rc = query_device(device, di);
  if (rc != TSB_OK) return rc;
  if (!di.coop) return TSB_EUNSUPPORTED;
  tsb::RoundsSync* sy = nullptr;
  uint4* scratch = nullptr;
  long long* d_out = nullptr;
  int grid = std::min(di.sms, tsb::LL_MAX_SMS);
  if (ctas > 0 && ctas < grid) grid = ctas;
  TSB_CUDA(cudaMalloc(&sy, sizeof(*sy)));
  const size_t scratch_bytes = std::max<size_t>((static_cast<size_t>(grid) * tsb::LL_T + 2) * sizeof(uint4), 2 * 256 * 256 * 4);
  TSB_CUDA(cudaMalloc(&scratch, scratch_bytes));
  TSB_CUDA(cudaMemset(scratch, 0, scratch_bytes));
  TSB_CUDA(cudaMalloc(&d_out, sizeof(long long)));
  TSB_CUDA(cudaMemset(sy, 0, sizeof(*sy)));
  unsigned epoch0 = 0;
  void* args[] = {&sy, &epoch0, &rounds, &variant, &scratch, &d_out};
  cudaError_t e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(tsb::rounds_sync_bench_kernel), dim3(grid),
                                              dim3(tsb::LL_T), args, 0, nullptr);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  long long cyc = 0;
  if (e == cudaSuccess) e = cudaMemcpy(&cyc, d_out, sizeof(cyc), cudaMemcpyDeviceToHost);
  cudaFree(sy);
  cudaFree(scratch);
  cudaFree(d_out);
  if (e != cudaSuccess) {
    g_last_cuda_error = std::string("flag exchange bench: ") + cudaGetErrorString(e);
    (void)cudaGetLastError();
    return TSB_ECUDA;
  }
  *cycles_per_round = static_cast<double>(cyc) / rounds;
  return TSB_OK;
}

// ---------------------------------------------------------------- N-Queens
static int nq_create(tsb_nq** out, int device, bool wide, int N, int g, int M_max) {
  if (!out || N < 1 || N > (wide ? TSB_MAX_QUEENS_WIDE : TSB_MAX_QUEENS) || g < 1 || M_max < 1) return TSB_EINVAL;
  tsb_nq* h = new (std::nothrow) tsb_nq();
  if (!h) return TSB_ENOMEM;
  h->N = N;
  h->g = g;
  h->wide = wide;
  if (const char* v = std::getenv("TSB200_NQ_TILE_THREADS")) h->tile_threads = std::atoi(v);
  const size_t rec = wide ? sizeof(tsb_nq_node24) : sizeof(tsb_nq_node);
  // (the arena starts with room for four worst-case rounds: every slot of every parent survives)
  h->pool.set_format(rec, tsb::NQ_TILE, 1, N, std::max<long long>(1LL << 22, 4LL * M_max * N));
  int rc = h->init(device, M_max, rec, static_cast<size_t>(N));
  if (rc != TSB_OK) {
    destroy(h);
    return rc;
  }
  *out = h;
  return TSB_OK;
}
int tsb_nq_create(tsb_nq** out, int device, int N, int g, int M_max) { return nq_create(out, device, false, N, g, M_max); }
int tsb_nq_create_wide(tsb_nq** out, int device, int max_queens, int N, int g, int M_max) {
  if (max_queens != TSB_MAX_QUEENS_WIDE) return TSB_EINVAL;
  return nq_create(out, device, true, N, g, M_max);
}

void tsb_nq_destroy(tsb_nq* h) { destroy(h); }

// ---- fused evaluate + generate_children, and the device-resident pool (SURVEY §8f rows 1, 3)
int tsb_nq_expand_device(tsb_nq* h, const void* parents_d, int count, void* children_d, uint64_t* n_children,
                         uint64_t* n_solutions, void* stream) {
  if (!h || count < 0 || !n_children || !n_solutions) return TSB_EINVAL;
  *n_children = *n_solutions = 0;
  if (count == 0) return TSB_OK;
  if (!parents_d || !children_d) return TSB_EINVAL;
  if (reinterpret_cast<uintptr_t>(parents_d) & 15) return TSB_EALIGN;
  TSB_CUDA(cudaSetDevice(h->device));
  unsigned long long nc = 0, ns = 0;
  const std::vector<PoolExtent> pieces{{0, count}};
  int rc = nq_expand(h, static_cast<const uint8_t*>(parents_d), pieces, static_cast<uint8_t*>(children_d),
                     stream ? static_cast<cudaStream_t>(stream) : h->stream, &nc, &ns);
  *n_children = nc;
  *n_solutions = ns;
  return rc;
}

int tsb_nq_expand(tsb_nq* h, const void* parents, int count, void* children, uint64_t capacity, uint64_t* n_children,
                  uint64_t* n_solutions) {
  if (!h || count < 0 || count > h->M_max || !n_children || !n_solutions) return TSB_EINVAL;
  *n_children = *n_solutions = 0;
  if (count == 0) return TSB_OK;
  if (!parents || !children) return TSB_EINVAL;
  return expand_host(*h, parents, count, children, capacity, n_children, n_solutions,
                     [h](auto arena, const auto& pieces, auto kids, auto nc, auto ns) {
                       return nq_expand(h, arena, pieces, kids, h->stream, nc, ns);
                     });
}

int tsb_nq_pool_push(tsb_nq* h, const void* nodes, int64_t n) {
  if (!h || n < 0 || (n && !nodes)) return TSB_EINVAL;
  if (!nq_nodes_valid(h->N, h->pool.rec, static_cast<const uint8_t*>(nodes), n)) return TSB_EINVAL;
  return pool_push(*h, nodes, n, [h] { return nq_materialize(h); });
}

int64_t tsb_nq_pool_size(const tsb_nq* h) { return pool_size(h); }

int tsb_nq_pool_step(tsb_nq* h, int m, int M, int64_t* n_parents, uint64_t* n_children, uint64_t* n_solutions) {
  if (!h || m < 1 || M < 1 || M > h->M_max || !n_parents || !n_children || !n_solutions) return TSB_EINVAL;
  return pool_step(*h, m, M, n_parents, n_children, n_solutions, [h] { return nq_materialize(h); },
                   [h](auto arena, const auto& pieces, auto kids, auto nc, auto ns) {
                     return nq_expand(h, arena, pieces, kids, h->stream, nc, ns, /*early=*/true);
                   });
}

int tsb_nq_pool_run(tsb_nq* h, int m, int M, int64_t max_rounds, uint64_t* n_rounds, uint64_t* n_parents,
                    uint64_t* n_children, uint64_t* n_solutions) {
  if (!h || m < 1 || M < 1 || M > h->M_max || max_rounds < 0 || !n_rounds || !n_parents || !n_children || !n_solutions)
    return TSB_EINVAL;
  return pool_run(NqRounds{}, h, m, M, max_rounds, n_rounds, n_parents, n_children, n_solutions);
}

int tsb_nq_sibling(tsb_nq* h, int index, tsb_nq** sibling) {
  return sibling_of(h, index, sibling, [h](tsb_nq** s) { return nq_create(s, h->device, h->wide, h->N, h->g, h->M_max); });
}

int tsb_nq_pools_per_launch(const tsb_nq* h, int M) {
  if (!h || M < 1 || M > h->M_max) return 1;
  return pools_per_launch(NqRounds{}, h, M);
}

int tsb_nq_pool_run_multi(tsb_nq* const* handles, int n_pools, int m, int M, int64_t max_rounds, uint64_t* out) {
  if (!handles || n_pools < 1 || n_pools > tsb::LL_MAX_POOLS || m < 1 || M < 1 || max_rounds < 0 || !out) return TSB_EINVAL;
  if (!one_group(handles, n_pools, M, [](const tsb_nq& h, const tsb_nq& h0) { return h.N == h0.N && h.wide == h0.wide; }))
    return TSB_EINVAL;
  return pool_run_multi(NqRounds{}, handles, n_pools, m, M, max_rounds, out);
}

int tsb_nq_pool_steal(tsb_nq* victim, tsb_nq* thief, int m, int64_t* n_stolen) {
  if (!victim || !thief || victim == thief || m < 1 || !n_stolen || victim->N != thief->N || victim->wide != thief->wide)
    return TSB_EINVAL;
  return pool_steal(*victim, *thief, m, n_stolen, [victim, thief] {
    const int rc = nq_materialize(victim);
    return rc == TSB_OK ? nq_materialize(thief) : rc;
  });
}

int tsb_nq_pool_drain(tsb_nq* h, void* nodes, int64_t capacity, int64_t* n) {
  if (!h || !n || capacity < 0) return TSB_EINVAL;
  return pool_drain(*h, nodes, capacity, n, [h] { return nq_materialize(h); });
}

int tsb_nq_evaluate(tsb_nq* h, const void* parents, int count, uint8_t* labels) {
  if (!h || count < 0 || count > h->M_max) return TSB_EINVAL;
  if (count == 0) return TSB_OK;
  if (!parents || !labels) return TSB_EINVAL;
  TSB_CUDA(cudaSetDevice(h->device));
  return h->evaluate_host(parents, count, labels, [h](const uint8_t* in, uint8_t* out, int n, cudaStream_t s) {
    return launch_nq(h, in, out, n, s);
  });
}

int tsb_nq_evaluate_device(tsb_nq* h, const void* parents_d, int count, uint8_t* labels_d, void* stream) {
  if (!h || count < 0) return TSB_EINVAL;
  if (count == 0) return TSB_OK;
  if (!parents_d || !labels_d) return TSB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(parents_d) | reinterpret_cast<uintptr_t>(labels_d)) & 15) return TSB_EALIGN;
  TSB_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : h->stream;
  return launch_nq(h, static_cast<const uint8_t*>(parents_d), labels_d, count, s);
}

int tsb_nq_register_host(tsb_nq* h, void* ptr, size_t bytes) { return register_host(h, ptr, bytes); }
int tsb_nq_unregister_host(tsb_nq* h, void* ptr) { return unregister_host(h, ptr); }
int tsb_nq_set_xfer(tsb_nq* h, int mode) { return set_xfer(h, mode); }
int tsb_nq_last_xfer(const tsb_nq* h) { return last_xfer(h); }
uint64_t tsb_nq_kernel_launches(const tsb_nq* h) { return kernel_launches(h); }
void* tsb_nq_stream(const tsb_nq* h) { return stream_of(h); }
int tsb_nq_max_queens(const tsb_nq* h) {
  if (!h) return TSB_EINVAL;
  return h->wide ? TSB_MAX_QUEENS_WIDE : TSB_MAX_QUEENS;
}

// ---------------------------------------------------------------- PFSP
int tsb_pfsp_create(tsb_pfsp** out, int device, int jobs, int machines, int M_max, const int32_t* p_times,
                    const int32_t* min_heads, const int32_t* min_tails, int nb_pairs, const int32_t* johnson,
                    const int32_t* lags, const int32_t* mp0, const int32_t* mp1, const int32_t* mp_order) {
  return tsb_pfsp_create_wide(out, device, TSB_MAX_JOBS, jobs, machines, M_max, p_times, min_heads, min_tails, nb_pairs,
                              johnson, lags, mp0, mp1, mp_order);
}

// The reference built with MAX_JOBS = max_jobs (lib/pfsp/PFSP_node.chpl:7): 20 = tsb_pfsp_create; 50 = 208-byte nodes,
// jobs == 50 instances (ta031..ta060), evaluated by the general kernels of pfsp_wide.cuh.  The exported expand, pool,
// sibling and run_multi entry points refuse such a handle (TSB_EUNSUPPORTED); the 50-job searches of tsb_host.cpp reach
// its device pool (pfsp_wide_expand.cuh) through the library-internal functions of pfsp_search_pool.h.
int tsb_pfsp_create_wide(tsb_pfsp** out, int device, int max_jobs, int jobs, int machines, int M_max, const int32_t* p_times,
                         const int32_t* min_heads, const int32_t* min_tails, int nb_pairs, const int32_t* johnson,
                         const int32_t* lags, const int32_t* mp0, const int32_t* mp1, const int32_t* mp_order) {
  if (!out || !p_times || !min_heads || !min_tails || M_max < 1 || nb_pairs < 0) return TSB_EINVAL;
  if (nb_pairs > 0 && (!johnson || !lags || !mp0 || !mp1 || !mp_order)) return TSB_EINVAL;
  if ((max_jobs != TSB_MAX_JOBS && max_jobs != TSB_MAX_JOBS_WIDE) || jobs != max_jobs || machines < 1 ||
      machines > TSB_MAX_MACHINES || nb_pairs > TSB_MAX_PAIRS)
    return TSB_EUNSUPPORTED;
  return pfsp_open(device, M_max,
                   pfsp_pack(max_jobs, jobs, machines, p_times, min_heads, min_tails, nb_pairs, johnson, lags, mp0, mp1,
                             mp_order),
                   out);
}

void tsb_pfsp_destroy(tsb_pfsp* h) { destroy(h); }

int tsb_pfsp_evaluate(tsb_pfsp* h, int lb_kind, const void* parents, int count, int64_t best, int32_t* bounds) {
  if (int rc = pfsp_check(h, false, lb_kind); rc != TSB_OK) return rc;
  if (count < 0 || count > h->M_max) return TSB_EINVAL;
  if (count == 0) return TSB_OK;
  if (!parents || !bounds) return TSB_EINVAL;
  TSB_CUDA(cudaSetDevice(h->device));
  return h->evaluate_host(parents, count, bounds,
                          [h, lb_kind, best](const uint8_t* in, uint8_t* out, int n, cudaStream_t s) {
                            return launch_pfsp(h, lb_kind, in, out, n, best, s);
                          });
}

int tsb_pfsp_evaluate_device(tsb_pfsp* h, int lb_kind, const void* parents_d, int count, int64_t best,
                             int32_t* bounds_d, void* stream) {
  if (int rc = pfsp_check(h, false, lb_kind); rc != TSB_OK) return rc;
  if (count < 0) return TSB_EINVAL;
  if (count == 0) return TSB_OK;
  if (!parents_d || !bounds_d) return TSB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(parents_d) | reinterpret_cast<uintptr_t>(bounds_d)) & 15) return TSB_EALIGN;
  TSB_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : h->stream;
  return launch_pfsp(h, lb_kind, static_cast<const uint8_t*>(parents_d), reinterpret_cast<uint8_t*>(bounds_d),
                     count, best, s);
}

int tsb_pfsp_register_host(tsb_pfsp* h, void* ptr, size_t bytes) { return register_host(h, ptr, bytes); }
int tsb_pfsp_unregister_host(tsb_pfsp* h, void* ptr) { return unregister_host(h, ptr); }
int tsb_pfsp_set_xfer(tsb_pfsp* h, int mode) { return set_xfer(h, mode); }
int tsb_pfsp_last_xfer(const tsb_pfsp* h) { return last_xfer(h); }
uint64_t tsb_pfsp_kernel_launches(const tsb_pfsp* h) { return kernel_launches(h); }
void* tsb_pfsp_stream(const tsb_pfsp* h) { return stream_of(h); }

uint64_t tsb_pfsp_slow_rounds(const tsb_pfsp* h) { return h ? h->slow_rounds : 0; }

int tsb_pfsp_route(const tsb_pfsp* h) {
  if (!h) return TSB_EINVAL;
  const PfspPacked& t = *h->tab;
  return t.mt | (t.simd16 ? TSB_ROUTE_SIMD16 : 0) | (t.pairs > 0 ? TSB_ROUTE_LB2 : 0) | (t.lb2u ? TSB_ROUTE_LB2U : 0);
}

int tsb_pfsp_expand_device(tsb_pfsp* h, int lb_kind, const void* parents_d, int count, int64_t* best,
                           void* children_d, uint64_t* n_children, uint64_t* n_solutions, void* stream) {
  if (int rc = pfsp_check(h, true, lb_kind); rc != TSB_OK) return rc;
  if (count < 0 || !best || !n_children || !n_solutions) return TSB_EINVAL;
  *n_children = *n_solutions = 0;
  if (count == 0) return TSB_OK;
  if (!parents_d || !children_d || count > h->M_max) return TSB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(parents_d) & 15) || (reinterpret_cast<uintptr_t>(children_d) & 7)) return TSB_EALIGN;
  TSB_CUDA(cudaSetDevice(h->device));
  unsigned long long nc = 0, ns = 0;
  const std::vector<PoolExtent> pieces{{0, count}};
  int rc = pfsp_expand_round(h, lb_kind, static_cast<const uint8_t*>(parents_d), pieces,
                             static_cast<uint8_t*>(children_d), stream ? static_cast<cudaStream_t>(stream) : h->stream,
                             best, &nc, &ns);
  *n_children = nc;
  *n_solutions = ns;
  return rc;
}

int tsb_pfsp_expand(tsb_pfsp* h, int lb_kind, const void* parents, int count, int64_t* best, void* children,
                    uint64_t capacity, uint64_t* n_children, uint64_t* n_solutions) {
  if (int rc = pfsp_check(h, true, lb_kind); rc != TSB_OK) return rc;
  if (count < 0 || count > h->M_max || !best || !n_children || !n_solutions) return TSB_EINVAL;
  *n_children = *n_solutions = 0;
  if (count == 0) return TSB_OK;
  if (!parents || !children) return TSB_EINVAL;
  return expand_host(*h, parents, count, children, capacity, n_children, n_solutions,
                     [h, lb_kind, best](auto arena, const auto& pieces, auto kids, auto nc, auto ns) {
                       return pfsp_expand_round(h, lb_kind, arena, pieces, kids, h->stream, best, nc, ns);
                     });
}

int tsb_pfsp_pool_push(tsb_pfsp* h, const void* nodes, int64_t n) {
  if (int rc = pfsp_check(h, true); rc != TSB_OK) return rc;
  if (n < 0 || (n && !nodes)) return TSB_EINVAL;
  return pool_push(*h, nodes, n, pfsp_plain);
}

int64_t tsb_pfsp_pool_size(const tsb_pfsp* h) { return pool_size(h); }

int tsb_pfsp_pool_step(tsb_pfsp* h, int lb_kind, int m, int M, int64_t* best, int64_t* n_parents,
                       uint64_t* n_children, uint64_t* n_solutions) {
  if (int rc = pfsp_check(h, true, lb_kind); rc != TSB_OK) return rc;
  if (m < 1 || M < 1 || M > h->M_max || !best || !n_parents || !n_children || !n_solutions) return TSB_EINVAL;
  return pfsp_step(h, lb_kind, m, M, best, n_parents, n_children, n_solutions);
}

int tsb_pfsp_pool_steal(tsb_pfsp* victim, tsb_pfsp* thief, int m, int64_t* n_stolen) {
  if (!victim || !thief || victim == thief || m < 1 || !n_stolen || victim->tab->jobs != thief->tab->jobs) return TSB_EINVAL;
  return pool_steal(*victim, *thief, m, n_stolen, pfsp_plain);
}

int tsb_pfsp_pool_drain(tsb_pfsp* h, void* nodes, int64_t capacity, int64_t* n) {
  if (!h || !n || capacity < 0) return TSB_EINVAL;
  return pool_drain(*h, nodes, capacity, n, pfsp_plain);
}

int tsb_pfsp_pool_run(tsb_pfsp* h, int lb_kind, int m, int M, int64_t max_rounds, int64_t* best, uint64_t* n_rounds,
                      uint64_t* n_parents, uint64_t* n_children, uint64_t* n_solutions) {
  if (int rc = pfsp_check(h, true, lb_kind); rc != TSB_OK) return rc;
  if (m < 1 || M < 1 || M > h->M_max || max_rounds < 0 || !best || !n_rounds || !n_parents || !n_children || !n_solutions)
    return TSB_EINVAL;
  return pool_run(PfspRounds{lb_kind, best}, h, m, M, max_rounds, n_rounds, n_parents, n_children, n_solutions);
}

int tsb_pfsp_sibling(tsb_pfsp* h, int index, tsb_pfsp** sibling) {
  if (int rc = pfsp_check(h, true); rc != TSB_OK) return rc;
  return sibling_of(h, index, sibling, [h](tsb_pfsp** s) { return pfsp_open(h->device, h->M_max, h->tab, s); });
}

int tsb_pfsp_pools_per_launch(const tsb_pfsp* h, int lb_kind, int M) {
  if (pfsp_check(h, true) != TSB_OK || M < 1 || M > h->M_max) return 1;
  if (cudaSetDevice(h->device) != cudaSuccess) {
    (void)cudaGetLastError();
    return 1;
  }
  // (const: what the occupancy query caches on the handle does not change what it computes)
  return pools_per_launch(PfspRounds{lb_kind, nullptr}, const_cast<tsb_pfsp*>(h), M);
}

int tsb_pfsp_pool_run_multi(tsb_pfsp* const* handles, int n_pools, int lb_kind, int m, int M, int64_t max_rounds,
                            int64_t* best, uint64_t* out) {
  if (!handles || n_pools < 1 || n_pools > tsb::PFR_MAX_POOLS || lb_kind < 0 || lb_kind > 2 || m < 1 || M < 1 ||
      max_rounds < 0 || !best || !out)
    return TSB_EINVAL;
  for (int i = 0; i < n_pools; i++)
    if (int rc = pfsp_check(handles[i], true); rc != TSB_OK) return rc;
  if (!one_group(handles, n_pools, M,
                 [](const tsb_pfsp& h, const tsb_pfsp& h0) { return tsb_pfsp_route(&h) == tsb_pfsp_route(&h0); }))
    return TSB_EINVAL;
  if (int rc = pfsp_check(handles[0], true, lb_kind); rc != TSB_OK) return rc;
  return pool_run_multi(PfspRounds{lb_kind, best}, handles, n_pools, m, M, max_rounds, out);
}

}  // extern "C"

// ============================================================================ library-internal (pfsp_search_pool.h)
namespace tsb::search {

int pfsp_pool_push(tsb_pfsp* h, const void* nodes, int64_t n) {
  if (!h || !h->tab->wide) return tsb_pfsp_pool_push(h, nodes, n);
  if (n < 0 || (n && !nodes)) return TSB_EINVAL;
  return pool_push(*h, nodes, n, pfsp_plain);
}

int pfsp_sibling(tsb_pfsp* h, int index, tsb_pfsp** sibling) {
  if (!h || !h->tab->wide) return tsb_pfsp_sibling(h, index, sibling);
  return sibling_of(h, index, sibling, [h](tsb_pfsp** s) { return pfsp_open(h->device, h->M_max, h->tab, s); });
}

int pfsp_pool_run_multi(tsb_pfsp* const* handles, int n_pools, int lb_kind, int m, int M, int64_t max_rounds,
                        int64_t* best, uint64_t* out) {
  if (!handles || !handles[0] || !handles[0]->tab->wide)
    return tsb_pfsp_pool_run_multi(handles, n_pools, lb_kind, m, M, max_rounds, best, out);
  if (n_pools < 1 || n_pools > tsb::PFR_MAX_POOLS || m < 1 || M < 1 || max_rounds < 0 || !best || !out) return TSB_EINVAL;
  for (int i = 0; i < n_pools; i++)
    if (int rc = pfsp_check(handles[i], false, lb_kind); rc != TSB_OK) return rc;
  if (!one_group(handles, n_pools, M, [](const tsb_pfsp& h, const tsb_pfsp& h0) { return h.tab->wide == h0.tab->wide; }))
    return TSB_EINVAL;
  return pool_run_multi(PfspWideRounds{{lb_kind, best}}, handles, n_pools, m, M, max_rounds, out);
}

}  // namespace tsb::search

// libtsb200_cbase.so: evaluate_gpu of the reference's C+CUDA PFSP drivers (baselines/pfsp/lib/evaluate.h) on top of
// libtsb200.so (include/tsb200_cbase.h has the contract).  No kernel lives here: every call is one
// tsb_pfsp_evaluate_device on a handle built from the caller's tables.
#include <cuda_runtime.h>

#include <atomic>
#include <cstdio>
#include <map>
#include <mutex>
#include <thread>
#include <tuple>
#include <vector>

#include "tsb200.h"
#include "tsb200_cbase.h"

static_assert(sizeof(Node) == sizeof(tsb_pfsp_node), "Node must be the 88-byte record of tsb200.h");
static_assert(sizeof(lb1_bound_data) == 32 && sizeof(lb2_bound_data) == 56, "the reference's LP64 layouts");

namespace {

// What identifies one driver task's tables: the reference builds them once per task (per GPU in
// pfsp_multigpu_cuda.c) and never changes them during the search.
using Key = std::tuple<std::thread::id, int, const int*, const int*, const int*, const int*, const int*, const int*,
                       const int*, const int*, int, int, int>;

// A key's handle, or the code tsb_pfsp_create refused its tables with (so that a refused key is not copied again on
// every call).
struct Entry {
  tsb_pfsp* h = nullptr;
  int rc = TSB_OK;
};

std::mutex g_mu;
// Leaked on purpose: destroying handles from a static destructor would run after the CUDA runtime's own teardown.
std::map<Key, Entry>& cache() {
  static auto* m = new std::map<Key, Entry>();
  return *m;
}
std::atomic<int> g_status{TSB_OK};

// One line on stderr and the sticky status (the first code since load or the last release wins).
void fail(int rc, int jobs, int lb, int size, const char* what, const char* cuda_text) {
  int expected = TSB_OK;
  g_status.compare_exchange_strong(expected, rc);
  std::fprintf(stderr, "tsb200_cbase: evaluate_gpu(jobs=%d, lb=%d, size=%d): %s: %s (%d)%s%s\n", jobs, lb, size, what,
               tsb_strerror(rc), rc, cuda_text && *cuda_text ? " - " : "", cuda_text ? cuda_text : "");
}

// The caller's device tables copied to the host, then a handle with chunks of up to M_max parents on `device`.
int build_handle(int device, int M_max, const lb1_bound_data& l1, const lb2_bound_data& l2, tsb_pfsp** out,
                 const char** cuda_text) {
  const int jobs = l1.nb_jobs, machines = l1.nb_machines, pairs = l2.nb_machine_pairs;
  if (machines < 1 || machines > TSB_MAX_MACHINES || pairs < 0 || pairs > TSB_MAX_PAIRS) return TSB_EUNSUPPORTED;
  std::vector<int32_t> pt(static_cast<size_t>(machines) * jobs), heads(machines), tails(machines);
  std::vector<int32_t> js(static_cast<size_t>(pairs) * jobs), lags(js.size()), mp0(pairs), mp1(pairs), order(pairs);
  auto get = [cuda_text](std::vector<int32_t>& dst, const int* src) -> int {
    if (dst.empty()) return TSB_OK;
    const cudaError_t e = cudaMemcpy(dst.data(), src, dst.size() * sizeof(int32_t), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) return TSB_OK;
    (void)cudaGetLastError();
    *cuda_text = cudaGetErrorString(e);
    return TSB_ECUDA;
  };
  int rc = TSB_OK;
  for (auto [dst, src] : {std::pair{&pt, l1.p_times}, {&heads, l1.min_heads}, {&tails, l1.min_tails},
                          {&js, l2.johnson_schedules}, {&lags, l2.lags}, {&mp0, l2.machine_pairs_1},
                          {&mp1, l2.machine_pairs_2}, {&order, l2.machine_pair_order}})
    if (rc == TSB_OK) rc = get(*dst, src);
  if (rc != TSB_OK) return rc;
  return tsb_pfsp_create(out, device, jobs, machines, M_max, pt.data(), heads.data(), tails.data(), pairs, js.data(),
                         lags.data(), mp0.data(), mp1.data(), order.data());
}

}  // namespace

extern "C" {

void evaluate_gpu(const int jobs, const int lb, const int size, const int nbBlocks, int* best,
                  const lb1_bound_data lbound1, const lb2_bound_data lbound2, Node* parents, int* bounds) {
  (void)nbBlocks;
  if (jobs != TSB_MAX_JOBS) return fail(TSB_EUNSUPPORTED, jobs, lb, size, "jobs must be 20", nullptr);
  if (lb < TSB_LB1_D || lb > TSB_LB2 || size < 0 || size % jobs != 0 || lbound1.nb_jobs != jobs)
    return fail(TSB_EINVAL, jobs, lb, size, "arguments", nullptr);
  if (size == 0) return;
  if (!parents || !bounds || !lbound1.p_times || !lbound1.min_heads || !lbound1.min_tails || (lb == TSB_LB2 && !best))
    return fail(TSB_EINVAL, jobs, lb, size, "null pointer", nullptr);
  // lb2 tables are optional for lb1 / lb1_d callers: without all five pointers the handle has no machine pairs
  lb2_bound_data l2 = lbound2;
  const bool has_lb2 = l2.nb_machine_pairs > 0 && l2.johnson_schedules && l2.lags && l2.machine_pairs_1 &&
                       l2.machine_pairs_2 && l2.machine_pair_order;
  if (!has_lb2) l2 = lb2_bound_data{};
  else if (l2.nb_jobs != jobs || l2.nb_machines != lbound1.nb_machines)
    return fail(TSB_EINVAL, jobs, lb, size, "lb2 table sizes", nullptr);

  int device = 0;
  if (const cudaError_t e = cudaGetDevice(&device); e != cudaSuccess) {
    (void)cudaGetLastError();
    return fail(TSB_ENODEV, jobs, lb, size, "cudaGetDevice", cudaGetErrorString(e));
  }
  const int count = size / jobs;
  const Key key{std::this_thread::get_id(), device, lbound1.p_times, lbound1.min_heads, lbound1.min_tails,
                l2.johnson_schedules, l2.lags, l2.machine_pairs_1, l2.machine_pairs_2, l2.machine_pair_order,
                lbound1.nb_jobs, lbound1.nb_machines, l2.nb_machine_pairs};
  Entry e;
  const char* cuda_text = nullptr;
  {
    std::lock_guard<std::mutex> lock(g_mu);
    auto it = cache().find(key);
    if (it == cache().end()) {
      // (the first chunk's size as M_max only sizes the handle's host-route buffers, which this path never uses)
      Entry fresh;
      fresh.rc = build_handle(device, count, lbound1, l2, &fresh.h, &cuda_text);
      if (fresh.rc == TSB_ECUDA && !cuda_text) cuda_text = tsb_last_cuda_error();
      // a copy that failed is not the tables' fault: it is retried on the next call
      if (fresh.rc != TSB_ECUDA && fresh.rc != TSB_ENOMEM) it = cache().emplace(key, fresh).first;
      e = fresh;
    } else {
      e = it->second;
    }
  }
  if (e.rc != TSB_OK) return fail(e.rc, jobs, lb, size, "tables", cuda_text);
  // (handles are per thread, so the call below runs outside the lock; the key's thread is the only user of e.h)
  const int64_t b = lb == TSB_LB2 ? *best : INT32_MAX;
  const int rc = tsb_pfsp_evaluate_device(e.h, lb, parents, count, b, bounds, cudaStreamLegacy);
  if (rc != TSB_OK)
    return fail(rc, jobs, lb, size, lb == TSB_LB2 && !(tsb_pfsp_route(e.h) & TSB_ROUTE_LB2) ? "lb2 refused on these tables"
                                                                                             : "tsb_pfsp_evaluate_device",
                rc == TSB_ECUDA ? tsb_last_cuda_error() : nullptr);
}

int tsb_cbase_status(void) { return g_status.load(); }

void tsb_cbase_release(void) {
  std::lock_guard<std::mutex> lock(g_mu);
  for (auto& kv : cache())
    if (kv.second.h) tsb_pfsp_destroy(kv.second.h);
  cache().clear();
  g_status.store(TSB_OK);
}

}  // extern "C"

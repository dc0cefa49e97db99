// pfsp_search_pool.h — the PFSP device-pool calls of the searches in tsb_host.cpp.  On a 20-job handle each is the
// exported call of the same name (tsb_pfsp_pool_push, tsb_pfsp_sibling, tsb_pfsp_pool_run_multi).  On a 50-job handle
// (tsb_pfsp_create_wide), which those refuse with TSB_EUNSUPPORTED, each runs the same operation on the handle's
// 208-byte pool: for lb1 and lb1_d, launches of the persistent kernel of pfsp_wide_rounds.cuh that serve all the pools
// (one pool per launch, in turn, or the step loop, where pfw_takes does not take M); for lb2, rounds of
// pfsp_wide_expand.cuh, one pool after the other.
#pragma once
#include <cstdint>

#include "tsb200.h"

// (internal to libtsb200.so: none of it is exported)
#pragma GCC visibility push(hidden)
namespace tsb::search {

int pfsp_pool_push(tsb_pfsp* h, const void* nodes, int64_t n);
int pfsp_sibling(tsb_pfsp* h, int index, tsb_pfsp** sibling);
int pfsp_pool_run_multi(tsb_pfsp* const* handles, int n_pools, int lb_kind, int m, int M, int64_t max_rounds,
                        int64_t* best, uint64_t* out);

}  // namespace tsb::search
#pragma GCC visibility pop

// pfr_tiers.h — how large a chunk one launch of the persistent PFSP kernel (pfsp_rounds.cuh) takes per pool, as a
// function of the GPU's SM count and of the number of independent pools the launch serves.  Shared by the library
// (pfsp_rounds_grid, pfsp_multi_grid) and the tests, which compile it as plain C++: no CUDA here.
#pragma once

namespace tsb {

constexpr int PFR_SLICE = 384;      // parents per CTA and round (three 128-parent tiles)
constexpr int PFR_MAX_CTAS = 256;   // CTAs per pool at most (the slots of its exchanges, PfRoundsSync)
constexpr int PFR_MAX_POOLS = 4;    // independent pools one launch can serve (blockIdx.y)

// CTAs per pool when one launch serves `pools` pools: one pool: one CTA per SM; several: two CTAs per SM in all
constexpr int pf_ctas_per_pool(int sms, int pools) {
  const int most = pools <= 1 ? sms : 2 * sms / pools;
  return most < PFR_MAX_CTAS ? most : PFR_MAX_CTAS;
}
// largest chunk (parents) of each pool.  On a 132-SM H100: one pool or two: 50 688 (covers the reference's default
// --M 50000), three: 33 792, four: 25 344.  One pool alone takes the kernel only up to PFR_MAX_M as well, so above
// it a pool that a shared launch leaves running alone finishes in two-kernel rounds.
constexpr long long pf_pool_capacity(int sms, int pools) {
  return static_cast<long long>(pf_ctas_per_pool(sms, pools)) * PFR_SLICE;
}

// The persistent kernel of 50-job pools (pfsp_wide_rounds.cuh) has the same slice, so the same capacities.  What it
// takes is what tools/pfsp50_rounds.py measured faster than the step loop on an H100 (DESIGN §7): one pool up to its
// capacity (measured to 50 688), two pools sharing a launch up to M = 20 000 (measured to there), never three or four
// (not measured; their pools take the one-pool kernel in turn).
constexpr int PFW_MAX_M_ONE = 50688;
constexpr int PFW_MAX_M_SHARED = 20000;
constexpr int PFW_MAX_POOLS_SHARED = 2;
// whether one launch of that kernel takes `pools` pools with chunks of up to M parents (the occupancy of the kernel
// itself aside).  Taking K >= 2 pools implies taking any 2..K of them: the shared launch's pools leave it one by one.
constexpr bool pfw_takes(int sms, int pools, long long M) {
  return pools >= 1 && pools <= PFW_MAX_POOLS_SHARED && M <= pf_pool_capacity(sms, pools) &&
         M <= (pools == 1 ? PFW_MAX_M_ONE : PFW_MAX_M_SHARED);
}

}  // namespace tsb

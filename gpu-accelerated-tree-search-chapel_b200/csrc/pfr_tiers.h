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

}  // namespace tsb

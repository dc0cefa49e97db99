// ll_tiers.h — how large a chunk one launch of the persistent N-Queens kernel (nq_rounds_ll.cuh) takes, as a
// function of the GPU's SM count.  Shared by the library (nq_ll_grid) and the search drivers (tsb_host.cpp), which
// size the warm-up and the steal policy by it before any handle exists; and when a launch clears the 16-bit tags of
// the pool's arena first.  Plain C++: no CUDA here.
#pragma once

namespace tsb {

constexpr int LL_MAX_SMS = 256;  // CTAs per pool at most (the count slots of a launch, LlSync)
constexpr int LL_SLICE2 = 512;   // parents per CTA with two parents per thread (256 threads)
constexpr int LL_SLICE3 = 768;   // ... with three

// CTAs per pool when one launch serves `pools` pools: one pool: one CTA per SM; several: two pools' CTAs per SM in all
// (with four pools, as the two halves of one CTA: nq_rounds_ll_kernel)
constexpr int ll_ctas_per_pool(int sms, int pools) {
  return pools <= 1 ? (sms < LL_MAX_SMS ? sms : LL_MAX_SMS) : 2 * (sms < LL_MAX_SMS ? sms : LL_MAX_SMS) / pools;
}
// largest chunk (parents) of each pool: one pool runs the 512-parent build, several the 768-parent one
constexpr long long ll_pool_capacity(int sms, int pools) {
  return static_cast<long long>(ll_ctas_per_pool(sms, pools)) * (pools <= 1 ? LL_SLICE2 : LL_SLICE3);
}
// pools per launch the drivers use for chunks of up to M parents: 4, 3, 2 (up to the one-pool capacity), or 1
// (beyond it: two-kernel rounds).  On an H100 (132 SMs): 4 up to 50 688, 3 up to 67 584, then 1.
// (tsb_nq_pools_per_launch answers a different question, the most pools one launch can take: 4, 3, 2 up to
// ll_pool_capacity(sms, 2) = 101 376 on an H100, then 1.  Above the one-pool capacity, a pool that such a launch
// leaves running alone finishes in two-kernel rounds.  The drivers cap it by this function and TSB200_POOLS, so
// beyond the one-pool capacity they run one pool in two-kernel rounds.)
constexpr int ll_pools_for(int sms, long long M) {
  return M <= ll_pool_capacity(sms, 4) ? 4 : M <= ll_pool_capacity(sms, 3) ? 3 : M <= ll_pool_capacity(sms, 1) ? 2 : 1;
}

// epochs after a clear of the arena's tags that a launch may use (the tags of epochs repeat mod 65535; the argument
// is at the top of nq_rounds_ll.cuh)
constexpr unsigned LL_TAG_SPAN = 65535u;
// Before a launch at epoch `epoch` (the last one used) that may run `max_rounds` rounds, with the arena's tags last
// cleared at epoch `clear_epoch`: whether to clear them first (then the clear's epoch is `epoch`), and the last epoch
// the launch may use.  A launch that would have fewer than min(max_rounds, LL_TAG_SPAN / 2) epochs left clears, so
// a clear comes at most once per 32 767 rounds.
struct LlTagWindow {
  bool clear;
  unsigned epoch_last;
};
constexpr LlTagWindow ll_tag_window(unsigned epoch, unsigned clear_epoch, long long max_rounds) {
  const long long left = static_cast<long long>(clear_epoch) + LL_TAG_SPAN - epoch;
  const long long want = max_rounds < LL_TAG_SPAN / 2 ? max_rounds : LL_TAG_SPAN / 2;
  return left < want ? LlTagWindow{true, epoch + LL_TAG_SPAN} : LlTagWindow{false, clear_epoch + LL_TAG_SPAN};
}

}  // namespace tsb

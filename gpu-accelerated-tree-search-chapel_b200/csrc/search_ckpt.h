// search_ckpt.h — the checkpoint file of a resumable search, on device pools (tsb_*_search_device_ckpt) or on host
// pools (tsb_*_search_ckpt).  Only search_ckpt.cpp knows the file's layout; the search driver (tsb_host.cpp) fills and
// reads this state.
#pragma once
#include <cstdint>
#include <vector>

// (internal to libtsb200.so: none of it is exported)
#pragma GCC visibility push(hidden)
namespace tsb::ckpt {

enum Problem : uint32_t { kNQueens = 1, kPfsp = 2 };

// what a checkpoint must match to be resumed: problem, node record size (21 / 25 / 88 / 208 bytes) and the call's
// parameters (N-Queens: a = N, b = g, c = 0; PFSP: a = inst, b = lb_kind, c = ub; pools: device pools per task, 1..4
// for PFSP, 0 for N-Queens, whose device pools are counted per task).
// A host-pool search writes pools = 0, which no PFSP device-pool search has; an N-Queens host-pool search also writes
// c = 1, since its device-pool twin writes pools = 0 too.  Its every unfinished task holds exactly one pool state.
struct Params {
  uint32_t problem = 0, rec = 0;
  int32_t a = 0, b = 0, c = 0, m = 0, M = 0, D = 0, pools = 0;
  bool operator==(const Params& o) const {
    return problem == o.problem && rec == o.rec && a == o.a && b == o.b && c == o.c && m == o.m && M == o.M &&
           D == o.D && pools == o.pools;
  }
  bool host() const { return pools == 0 && (problem == kPfsp || c == 1); }
};

struct PoolState {  // one pool (device, or a host task's): its incumbent and its nodes in logical order (rec bytes each)
  int64_t best = 0;
  std::vector<uint8_t> nodes;
};

struct TaskState {  // one task of step 2: its counters so far
  uint64_t tree = 0, sol = 0, offloads = 0, parents = 0, launches = 0;
  int64_t best = 0;
  bool finished = false;      // it had left step 2 when the search stopped: `left` is its host pool, `pools` is empty
  std::vector<uint8_t> left;  // (front to back)
  std::vector<PoolState> pools;
};

struct State {
  Params p;
  uint64_t tree1 = 0, sol1 = 0;  // step 1
  int64_t best1 = 0;
  double t_step1 = 0, t_step2 = 0;  // t_step2: summed over the invocations so far
  uint64_t steals = 0;
  std::vector<TaskState> tasks;  // D entries
};

// 0: no file at `path`; 1: `st` holds the checkpoint; TSB_EINVAL: the file cannot be read, is damaged (size,
// checksum, magic, version; a host-pool task without exactly one pool state, or a finished one with any) or was
// written by another problem, node width or parameters than `want`.  Reads only.
int load(const char* path, const Params& want, State* st);
// writes `path`.tmp, fsyncs it and renames it over `path`: TSB_OK, or TSB_EINVAL if it cannot be written (an
// existing file at `path` is then unchanged)
int save(const char* path, const State& st);

}  // namespace tsb::ckpt
#pragma GCC visibility pop

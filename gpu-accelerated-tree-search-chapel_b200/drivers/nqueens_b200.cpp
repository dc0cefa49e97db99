// nqueens_b200 — C++ stand-in for nqueens_gpu_chpl / nqueens_multigpu_chpl (no Chapel compiler on the
// build and bench hosts).  Same CLI (--N --g --m --M --D, -h/--help; reference README.md:47-87,
// lib/commons/util.chpl:32-40), same defaults (nqueens_multigpu_chpl.chpl:19-23), same result lines
// (nqueens_gpu_chpl.chpl:39-46).  The search itself is tsb_nq_search in libtsb200.so, whose offload step
// is the C-ABI call a patched Chapel driver makes.
#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "tsb200.h"

// --checkpoint: SIGINT / SIGTERM stop the search at its next call boundary, and it writes the checkpoint
static void request_stop(int) { tsb_search_request_stop(); }
static void on_stop_signals() {
  struct sigaction sa;
  std::memset(&sa, 0, sizeof(sa));
  sa.sa_handler = request_stop;
  sigemptyset(&sa.sa_mask);
  sigaction(SIGINT, &sa, nullptr);
  sigaction(SIGTERM, &sa, nullptr);
}

int main(int argc, char** argv) {
  int N = 14, g = 1, m = 25, M = 50000, D = 1, devpool = 0;
  const char* ckpt = nullptr;
  double limit = -1;
  for (int i = 1; i < argc; i++) {
    if (!std::strcmp(argv[i], "-h") || !std::strcmp(argv[i], "--help")) {
      std::printf("\n  General Parameters:\n\n   --m   int   minimum number of elements to offload on a GPU device\n"
                  "   --M   int   maximum number of elements to offload on a GPU device\n"
                  "   --D   int   number of GPU device(s) (only in multi-GPU setting)\n"
                  "\n  N-Queens Benchmark Parameters:\n\n   --N   int   number of queens\n"
                  "   --g   int   number of safety check(s) per evaluation\n\n"
                  "  Device pools:\n\n   --devpool     int   1: the pool(s) of step 2 stay on the GPU(s)\n"
                  "   --checkpoint  str   (with --devpool 1) resumable search: continue from FILE if it exists; on a stop\n"
                  "                       (--time-limit, SIGINT, SIGTERM) write FILE and exit with 4; rerun the same\n"
                  "                       command to resume; FILE is removed when the search ends\n"
                  "   --time-limit  real  seconds of this run before it stops (0: after one call per task)\n\n");
      return 1;
    }
    if (i + 1 >= argc) break;
    if (!std::strcmp(argv[i], "--checkpoint")) {
      ckpt = argv[++i];
      continue;
    }
    if (!std::strcmp(argv[i], "--time-limit")) {
      limit = std::atof(argv[++i]);
      continue;
    }
    int* dst = !std::strcmp(argv[i], "--N") ? &N : !std::strcmp(argv[i], "--g") ? &g
             : !std::strcmp(argv[i], "--m") ? &m : !std::strcmp(argv[i], "--M") ? &M
             : !std::strcmp(argv[i], "--D") ? &D
             : !std::strcmp(argv[i], "--devpool") ? &devpool : nullptr;  // 1: pool of step 2 resident on the GPU
    if (dst) *dst = std::atoi(argv[++i]);
  }
  if (N <= 0 || g <= 0 || m <= 0 || M <= 0 || D <= 0) {
    std::fprintf(stderr, "All parameters must be positive integers.\n");
    return 2;
  }
  if ((ckpt || limit >= 0) && (!devpool || !ckpt)) {
    std::fprintf(stderr, "--checkpoint needs --devpool 1, and --time-limit needs --checkpoint.\n");
    return 2;
  }
  if (N > TSB_MAX_QUEENS_WIDE) {  // (N = 21..24 run as a `-sMAX_QUEENS=24` build would: 25-byte nodes)
    std::fprintf(stderr, "--N %d: boards of at most %d queens are supported.\n", N, TSB_MAX_QUEENS_WIDE);
    return 2;
  }
  std::printf("\n=================================================\n%s H100 (tsb200)\n\n"
              "Resolution of the %d-Queens instance\n  with %d safety check(s) per evaluation\n"
              "=================================================\n", D > 1 ? "Multi-GPU" : "Single-GPU", N, g);
  tsb_search_stats st;
  if (ckpt) on_stop_signals();
  const int rc = ckpt      ? tsb_nq_search_device_ckpt(TSB_MAX_QUEENS, N, g, m, M, D, ckpt, limit, &st)
                 : devpool ? tsb_nq_search_device(N, g, m, M, D, &st)
                           : tsb_nq_search(N, g, m, M, D, &st);
  if (rc == TSB_ESTOPPED) {
    std::printf("\nSearch stopped\nExplored so far: tree %llu, solutions %llu, %llu offloads, %f [s] on GPU\n"
                "checkpoint written to %s; rerun the same command to resume\n",
                (unsigned long long)st.explored_tree, (unsigned long long)st.explored_sol,
                (unsigned long long)st.offloads, st.t_step2, ckpt);
    return 4;
  }
  if (rc != TSB_OK) {
    std::fprintf(stderr, "tsb_nq_search: %s (%s)\n", tsb_strerror(rc), tsb_last_cuda_error());
    return 3;
  }
  std::printf("\nInitial search on CPU completed\nElapsed time: %f [s]\n\nSearch on GPU completed\n"
              "Elapsed time: %f [s]\n\nSearch on CPU completed\nElapsed time: %f [s]\n\nExploration terminated.\n",
              st.t_step1, st.t_step2, st.t_step3);
  if (D > 1) {  // shares of the step-2 tree, as nqueens_multigpu_chpl.chpl:337 divides (exploredTree - res1[1])
    uint64_t step2 = 0;
    for (int i = 0; i < D; i++) step2 += st.per_gpu_tree[i];
    std::printf("workload per GPU:");
    for (int i = 0; i < D; i++) std::printf(" %.2f", step2 ? 100.0 * st.per_gpu_tree[i] / (double)step2 : 0.0);
    std::printf("\nsteals between device pools: %llu\n", (unsigned long long)st.steals);
  }
  const double t = st.t_step1 + st.t_step2 + st.t_step3;
  std::printf("\n=================================================\n"
              "Size of the explored tree: %llu\nNumber of explored solutions: %llu\nElapsed time: %f [s]\n"
              "=================================================\n\n",
              (unsigned long long)st.explored_tree, (unsigned long long)st.explored_sol, t);
  std::printf("GPU diagnostics:\n   kernel_launch: %llu\n   offloads: %llu\n   Mnodes/s: %.2f\n",
              (unsigned long long)st.kernel_launches, (unsigned long long)st.offloads, st.explored_tree / t / 1e6);
  return 0;
}

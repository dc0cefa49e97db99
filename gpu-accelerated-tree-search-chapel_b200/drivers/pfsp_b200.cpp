// pfsp_b200 — C++ stand-in for pfsp_gpu_chpl / pfsp_multigpu_chpl.  Same CLI (--inst --lb --ub --m --M
// --D; README.md:47-87), same defaults (pfsp_multigpu_chpl.chpl:24-30: inst 14, lb "lb1", ub 1), same
// result lines (pfsp_gpu_chpl.chpl:66-77).  --lb takes the Chapel spelling lb1 | lb1_d | lb2.  --max-jobs 50 runs
// the program as the reference built with MAX_JOBS = 50 (lib/pfsp/PFSP_node.chpl:7): ta031..ta060.
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
  int inst = 14, ub = 1, m = 25, M = 50000, D = 1, lb = TSB_LB1, devpool = 0, pools = 1, max_jobs = TSB_MAX_JOBS;
  const char* lbs = "lb1";
  const char* ckpt = nullptr;
  double limit = -1;
  for (int i = 1; i < argc; i++) {
    if (!std::strcmp(argv[i], "-h") || !std::strcmp(argv[i], "--help")) {
      std::printf("\n  PFSP Benchmark Parameters:\n\n   --inst   int   Taillard's instance to solve (between 001 and 120)\n"
                  "   --lb     str   lower bound function (lb1, lb1_d, lb2)\n"
                  "   --ub     int   initial upper bound (0, 1)\n   --m --M --D as for N-Queens\n"
                  "   --devpool int  1: the pool(s) of step 2 stay on the GPU(s)\n"
                  "   --pools  int   device pools per GPU task (1..4; > 1 needs --devpool 1): each is one task\n"
                  "                  of the reference, with its own incumbent, sharing the GPU's launches\n"
                  "   --checkpoint str  (with --devpool 1) resumable search: continue from FILE if it exists; on a stop\n"
                  "                     (--time-limit, SIGINT, SIGTERM) write FILE and exit with 4; rerun the same\n"
                  "                     command to resume; FILE is removed when the search ends\n"
                  "   --time-limit real seconds of this run before it stops (0: after one call per task)\n"
                  "   --max-jobs int   MAX_JOBS of the build (20, 50): 50 solves ta031..ta060 on 208-byte nodes\n\n");
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
    if (!std::strcmp(argv[i], "--lb")) {
      lbs = argv[++i];
      lb = !std::strcmp(lbs, "lb1") ? TSB_LB1 : !std::strcmp(lbs, "lb1_d") ? TSB_LB1_D
           : !std::strcmp(lbs, "lb2") ? TSB_LB2 : -1;
      continue;
    }
    int* dst = !std::strcmp(argv[i], "--inst") ? &inst : !std::strcmp(argv[i], "--ub") ? &ub
             : !std::strcmp(argv[i], "--m") ? &m : !std::strcmp(argv[i], "--M") ? &M
             : !std::strcmp(argv[i], "--D") ? &D
             : !std::strcmp(argv[i], "--devpool") ? &devpool  // 1: pool(s) of step 2 resident on the GPU
             : !std::strcmp(argv[i], "--pools") ? &pools : !std::strcmp(argv[i], "--max-jobs") ? &max_jobs : nullptr;
    if (dst) *dst = std::atoi(argv[++i]);
  }
  if (m <= 0 || M <= 0) { std::fprintf(stderr, "Error: m and M must be positive integers.\n"); return 2; }
  if (pools < 1 || pools > 4 || (pools > 1 && !devpool)) {
    std::fprintf(stderr, "Error: --pools must be 1..4, and more than 1 needs --devpool 1\n");
    return 2;
  }
  if ((ckpt || limit >= 0) && (!devpool || !ckpt)) {
    std::fprintf(stderr, "Error: --checkpoint needs --devpool 1, and --time-limit needs --checkpoint\n");
    return 2;
  }
  if (inst < 1 || inst > 120) { std::fprintf(stderr, "Error: unsupported Taillard's instance\n"); return 2; }
  if (max_jobs != TSB_MAX_JOBS && max_jobs != TSB_MAX_JOBS_WIDE) {
    std::fprintf(stderr, "Error: --max-jobs must be %d or %d\n", TSB_MAX_JOBS, TSB_MAX_JOBS_WIDE);
    return 2;
  }
  if (lb < 0) { std::fprintf(stderr, "Error - Unsupported lower bound\n"); return 2; }
  if (ub != 0 && ub != 1) { std::fprintf(stderr, "Error: unsupported upper bound initialization\n"); return 2; }
  std::printf("\n=================================================\n%s H100 (tsb200)\n\n"
              "Resolution of PFSP Taillard's instance: ta%d (m = %d, n = %d)\nInitial upper bound: %s\n"
              "Lower bound function: %s\nBranching rule: fwd\n=================================================\n",
              D > 1 ? "Multi-GPU" : "Single-GPU", inst, tsb_taillard_nb_machines(inst), tsb_taillard_nb_jobs(inst),
              ub ? "opt" : "inf", lbs);
  tsb_search_stats st;
  if (ckpt) on_stop_signals();
  const bool wide = max_jobs == TSB_MAX_JOBS_WIDE;
  const int rc = wide ? (ckpt       ? tsb_pfsp_search_device_ckpt_wide(max_jobs, inst, lb, ub, m, M, D, pools, ckpt, limit, &st)
                         : !devpool ? tsb_pfsp_search_wide(max_jobs, inst, lb, ub, m, M, D, &st)
                                    : tsb_pfsp_search_device_wide(max_jobs, inst, lb, ub, m, M, D, pools, &st))
                 : ckpt      ? tsb_pfsp_search_device_ckpt(inst, lb, ub, m, M, D, pools, ckpt, limit, &st)
                 : !devpool  ? tsb_pfsp_search(inst, lb, ub, m, M, D, &st)
                 : pools > 1 ? tsb_pfsp_search_device_pools(inst, lb, ub, m, M, D, pools, &st)
                             : tsb_pfsp_search_device(inst, lb, ub, m, M, D, &st);
  if (rc == TSB_ESTOPPED) {
    std::printf("\nSearch stopped\nExplored so far: tree %llu, solutions %llu, best makespan %lld, %llu offloads, "
                "%f [s] on GPU\ncheckpoint written to %s; rerun the same command to resume\n",
                (unsigned long long)st.explored_tree, (unsigned long long)st.explored_sol, (long long)st.best,
                (unsigned long long)st.offloads, st.t_step2, ckpt);
    return 4;
  }
  if (rc != TSB_OK) {
    std::fprintf(stderr, "tsb_pfsp_search: %s (%s)\n", tsb_strerror(rc), tsb_last_cuda_error());
    return 3;
  }
  const double t = st.t_step1 + st.t_step2 + st.t_step3;
  std::printf("\nInitial search on CPU completed\nElapsed time: %f [s]\n\nSearch on GPU completed\n"
              "Elapsed time: %f [s]\n\nSearch on CPU completed\nElapsed time: %f [s]\n\nExploration terminated.\n",
              st.t_step1, st.t_step2, st.t_step3);
  if (D > 1) {  // shares of the step-2 tree (pfsp_multigpu_chpl.chpl:522)
    uint64_t step2 = 0;
    for (int i = 0; i < D; i++) step2 += st.per_gpu_tree[i];
    std::printf("workload per GPU:");
    for (int i = 0; i < D; i++) std::printf(" %.2f", step2 ? 100.0 * st.per_gpu_tree[i] / (double)step2 : 0.0);
    std::printf("\nsteals between device pools: %llu\n", (unsigned long long)st.steals);
  }
  const long long initUB = ub ? tsb_taillard_best_ub(inst) : 0x7fffffffffffffffLL;
  std::printf("\n=================================================\n"
              "Size of the explored tree: %llu\nNumber of explored solutions: %llu\n"
              "Optimal makespan: %lld%s\nElapsed time: %f [s]\n"
              "=================================================\n\n",
              (unsigned long long)st.explored_tree, (unsigned long long)st.explored_sol, (long long)st.best,
              st.best < initUB ? " (improved)" : " (not improved)", t);
  std::printf("GPU diagnostics:\n   kernel_launch: %llu\n   offloads: %llu\n   Mnodes/s: %.3f\n",
              (unsigned long long)st.kernel_launches, (unsigned long long)st.offloads, st.explored_tree / t / 1e6);
  return 0;
}

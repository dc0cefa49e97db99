/*
 * tsb_oracle.h — CPU ORACLE for the batch node-evaluation hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library, and only as the checker / CPU baseline.  The product
 * (libtsb200.so) never links, loads or calls it.
 *
 * It is a plain-C restatement of the reference's *Chapel* CPU path (Chapel is
 * authoritative where the reference's C baselines diverge, SURVEY.md Appendix A).
 * Every function cites the reference file:line it follows.
 *
 * Parity pinning: checked against (1) tests/golden/ vectors produced by the
 * reference's own C sources compiled into oracle/_ref (tests/golden/make_golden.py),
 * (2) the explored-tree / solution / optimum counts the reference binaries print
 * (SURVEY.md Appendix B) and (3) the classical N-Queens solution counts.
 */
#ifndef TSB_ORACLE_H
#define TSB_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OR_MAX_QUEENS 20   /* lib/nqueens/NQueens_node.chpl:7 */
#ifndef OR_MAX_JOBS
#define OR_MAX_JOBS 20     /* lib/pfsp/PFSP_node.chpl:7 (`config param MAX_JOBS`: oracle/Makefile builds a second \
                              library with -DOR_MAX_JOBS=50 = `chpl -sMAX_JOBS=50`, for ta031..ta060) */
#endif
#define OR_MAX_MACHINES 20 /* lib/pfsp/Bound_simple.chpl:3 (NUM_MACHINES) */

/* lib/nqueens/NQueens_node.chpl:9-11 — 21 bytes, align 1 */
typedef struct {
  uint8_t depth;
  uint8_t board[OR_MAX_QUEENS];
} or_nq_node;

/* lib/pfsp/PFSP_node.chpl:9-12 — 88 bytes (208 with MAX_JOBS = 50), align 4 */
typedef struct {
  int32_t depth;
  int32_t limit1;
  int32_t prmu[OR_MAX_JOBS];
} or_pfsp_node;

/* lb1_bound_data (Bound_simple.chpl:6-27) + lb2_bound_data (Bound_johnson.chpl:11-48) */
typedef struct {
  int32_t jobs, machines, pairs;
  int32_t p_times[OR_MAX_MACHINES * OR_MAX_JOBS]; /* machine-major: [k*jobs + job] */
  int32_t min_heads[OR_MAX_MACHINES];
  int32_t min_tails[OR_MAX_MACHINES];
  int32_t johnson[190 * OR_MAX_JOBS]; /* [pair*jobs + pos] -> job */
  int32_t lags[190 * OR_MAX_JOBS];    /* [pair*jobs + job] */
  int32_t mp0[190], mp1[190], mp_order[190];
} or_pfsp_tables;

/* ---- Taillard instances (lib/pfsp/Taillard.chpl) ---- */
int32_t or_taillard_nb_jobs(int id);
int32_t or_taillard_nb_machines(int id);
int64_t or_taillard_best_ub(int id);
void or_taillard_processing_times(int32_t* ptm, int id);

/* ---- table precompute; heads_mode 0 = Chapel semantics (authoritative), 1 = C-baseline semantics ---- */
int or_pfsp_tables_build(or_pfsp_tables* t, int inst, int heads_mode);
/* the same with one of the reference's lb2 variants (Bound_johnson.chpl:6, :36-43, :50-87): 0 LB2_FULL / 3 LB2_LEARN
 * (all pairs, what the reference compiles), 1 LB2_NABESHIMA (adjacent machines), 2 LB2_LAGEWEG (each machine with
 * the last one) */
int or_pfsp_tables_build_variant(or_pfsp_tables* t, int inst, int heads_mode, int variant);
/* the same precompute on a given machine-major matrix p_times[machines*jobs] (any values, any 1..OR_MAX_JOBS jobs
 * and 1..OR_MAX_MACHINES machines): 0, or -2 for dimensions out of range */
int or_pfsp_tables_from_ptimes(or_pfsp_tables* t, int jobs, int machines, const int32_t* p_times, int heads_mode,
                               int variant);

/* ---- bounds ---- */
int32_t or_eval_solution(const or_pfsp_tables* t, const int32_t* prmu);
int32_t or_lb1_bound(const or_pfsp_tables* t, const int32_t* prmu, int32_t limit1, int32_t limit2);
void or_lb1_children_bounds(const or_pfsp_tables* t, const int32_t* prmu, int32_t limit1, int32_t limit2,
                            int32_t* lb_begin /* [OR_MAX_JOBS] */);
int32_t or_lb2_bound(const or_pfsp_tables* t, const int32_t* prmu, int32_t limit1, int32_t limit2,
                     int64_t best);

/* ---- batch evaluators: write exactly the slots the reference kernels write ---- */
/* nqueens_gpu_chpl.chpl:97-123 */
void or_nq_evaluate(const or_nq_node* parents, int count, int N, int g, uint8_t* labels);
/* pfsp_gpu_chpl.chpl:192-270; lb_kind 0 = lb1_d, 1 = lb1, 2 = lb2 (encoding of baselines/pfsp/pfsp_c.c:86-88) */
void or_pfsp_evaluate(const or_pfsp_tables* t, int lb_kind, const or_pfsp_node* parents, int count,
                      int64_t best, int32_t* bounds);
/* same, over parents [begin, end) only — used by the threaded CPU baseline */
void or_nq_evaluate_range(const or_nq_node* parents, int begin, int end, int N, int g, uint8_t* labels);
void or_pfsp_evaluate_range(const or_pfsp_tables* t, int lb_kind, const or_pfsp_node* parents, int begin,
                            int end, int64_t best, int32_t* bounds);

/* evaluate_gpu + generate_children of one chunk (nqueens_gpu_chpl.chpl:97-149): children in the reference's
 * order; returns their number (children filled only if it fits `capacity`) */
int64_t or_nq_expand_chunk(const or_nq_node* parents, int count, int N, int g, or_nq_node* children,
                           int64_t capacity, uint64_t* solutions);

/* evaluate_gpu + generate_children of one PFSP chunk (pfsp_gpu_chpl.chpl:384-392, 273-303); *best is read at
 * entry (value at launch for the bounds) and lowered by the leaves in the reference's sequential order */
int64_t or_pfsp_expand_chunk(const or_pfsp_tables* t, int lb_kind, const or_pfsp_node* parents, int count,
                             int64_t* best, or_pfsp_node* children, int64_t capacity, uint64_t* solutions);

/* ---- whole searches ---- */
typedef struct {
  uint64_t tree, sol;
  int64_t best;
  uint64_t offloads, offloaded_parents, live_slots;
  uint64_t depth_hist[OR_MAX_JOBS + 2];
  double seconds;
  /* step 2 of each task of the D-way split (the reference's eachExploredTree / eachExploredSol, and the task's
   * best_l when step 2 ends); task 0 alone for D = 1 */
  uint64_t task_tree[8], task_sol[8];
  int64_t task_best[8];
} or_search_result;

/* nqueens_chpl.chpl:92-113 (sequential DFS) */
void or_nq_search_seq(int N, int g, or_search_result* r);
void or_nq_search_from(int N, int g, const or_nq_node* nodes, int n, uint64_t* tree, uint64_t* sol);
int or_nq_frontier(int N, int g, int depth, or_nq_node* out, int cap, uint64_t* tree, uint64_t* sol);
/* nqueens_gpu_chpl.chpl:152-248 / nqueens_multigpu_chpl.chpl:158-352 with the oracle as evaluator;
 * D >= 1 emulates the static strided split (no work stealing) sequentially, task after task (D <= 8). */
void or_nq_search_offload(int N, int g, int m, int M, int D, or_search_result* r);
/* pfsp_chpl.chpl:191-215 */
void or_pfsp_search_seq(int inst, int lb_kind, int ub, int heads_mode, or_search_result* r);
/* pfsp_gpu_chpl.chpl:306-431 / pfsp_multigpu_chpl.chpl with the oracle as evaluator */
void or_pfsp_search_offload(int inst, int lb_kind, int ub, int m, int M, int D, int heads_mode,
                            or_search_result* r);
/* one task `part` (0 <= part < D) of those searches run alone, as one process of a process-per-GPU launch runs it:
 * the same step 1 (credited to part 0 only) and static split, then step 2 of task `part` only, and step 3 on that
 * task's own leftovers with that task's own best.  The N-Queens step 1 grows the pool to `warm` nodes (D * m in the
 * reference; more when a task keeps several pools). */
void or_nq_search_offload_part(int N, int g, int m, int M, int D, int part, int warm, or_search_result* r);
void or_pfsp_search_offload_part(int inst, int lb_kind, int ub, int m, int M, int D, int part, int heads_mode,
                                 or_search_result* r);

/* capture the parents of offload number `which` (0-based) of the single-GPU N-Queens / PFSP driver
 * into out (capacity cap nodes); returns the chunk size or -1 */
int or_nq_capture_chunk(int N, int g, int m, int M, int which, or_nq_node* out, int cap);
int or_pfsp_capture_chunk(int inst, int lb_kind, int ub, int m, int M, int which, or_pfsp_node* out,
                          int cap, int64_t* best_at_launch);

#ifdef __cplusplus
}
#endif
#endif

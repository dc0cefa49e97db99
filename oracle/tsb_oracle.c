/*
 * tsb_oracle.c — CPU ORACLE (test infrastructure, NOT product code; see tsb_oracle.h).
 *
 * Plain-C restatement of the reference's Chapel CPU path for the batch node-evaluation
 * hot path: N-Queens conflict check and PFSP lb1 / lb1_d / lb2, the table precompute
 * they consume, and the sequential / offload search drivers whose printed counts pin
 * parity.  Each function cites the reference lines it follows (paths relative to the
 * reference root).  Written for clarity, not speed.
 */
#define _POSIX_C_SOURCE 200809L
#include "tsb_oracle.h"

#include <limits.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "taillard_data.inc"

#define OR_MAX(a, b) ((a) > (b) ? (a) : (b))
#define OR_MIN(a, b) ((a) < (b) ? (a) : (b))

static double now_s(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

/* ======================================================================== Taillard */

/* lib/pfsp/Taillard.chpl:29-36 */
int32_t or_taillard_nb_jobs(int id) {
  if (id > 110) return 500;
  if (id > 90) return 200;
  if (id > 60) return 100;
  if (id > 30) return 50;
  return 20;
}

/* lib/pfsp/Taillard.chpl:38-52 */
int32_t or_taillard_nb_machines(int id) {
  if (id > 110) return 20;
  if (id > 100) return 20;
  if (id > 90) return 10;
  if (id > 80) return 20;
  if (id > 70) return 10;
  if (id > 60) return 5;
  if (id > 50) return 20;
  if (id > 40) return 10;
  if (id > 30) return 5;
  if (id > 20) return 20;
  if (id > 10) return 10;
  return 5;
}

/* lib/pfsp/Taillard.chpl:54-70 */
int64_t or_taillard_best_ub(int id) { return TAILLARD_BEST_UB[id - 1]; }

/* lib/pfsp/Taillard.chpl:72-84 — Lehmer LCG with Schrage's trick; the 0..1 value is a
 * double division in Chapel (`seed:real / m:real`), float in the C baseline; SURVEY
 * Appendix A.(iii): identical outputs on all 120 instances. */
static int64_t taillard_unif(int64_t* seed, int64_t low, int64_t high) {
  const int64_t m = 2147483647, a = 16807, b = 127773, c = 2836;
  int64_t k = *seed / b;
  *seed = a * (*seed % b) - k * c;
  if (*seed < 0) *seed += m;
  double v01 = (double)*seed / (double)m;
  return low + (int64_t)(v01 * (double)(high - low + 1));
}

/* lib/pfsp/Taillard.chpl:86-97 — machine-major ptm[i*N + j] */
void or_taillard_processing_times(int32_t* ptm, int id) {
  const int N = or_taillard_nb_jobs(id), M = or_taillard_nb_machines(id);
  int64_t seed = TAILLARD_SEEDS[id - 1];
  for (int i = 0; i < M; i++)
    for (int j = 0; j < N; j++) ptm[i * N + j] = (int32_t)taillard_unif(&seed, 1, 99);
}

/* ======================================================================== tables */

/* lib/pfsp/Bound_simple.chpl:254-289.  heads_mode 0 reproduces the Chapel statement
 * `data.min_heads[k] = min(max(int(32)), tmp0)` (:271), which OVERWRITES min_heads[k]
 * with the current job's head, so after the job loop it holds the heads of the LAST
 * job (SURVEY Appendix A.1).  heads_mode 1 is the C baseline's true minimum
 * (baselines/pfsp/lib/c_bound_simple.c:300), kept only to cross-check against _ref. */
static void fill_min_heads_tails(or_pfsp_tables* t, int heads_mode) {
  const int N = t->jobs, M = t->machines;
  const int32_t* p = t->p_times;
  int32_t tmp0, tmp1;

  for (int k = 0; k < M; k++) t->min_heads[k] = INT32_MAX;
  t->min_heads[0] = 0;
  for (int i = 0; i < N; i++) {
    tmp0 = p[i];
    for (int k = 1; k < M; k++) {
      tmp1 = tmp0 + p[k * N + i];
      if (heads_mode == 0)
        t->min_heads[k] = OR_MIN(INT32_MAX, tmp0);
      else
        t->min_heads[k] = OR_MIN(t->min_heads[k], tmp0);
      tmp0 = tmp1;
    }
  }

  for (int k = 0; k < M; k++) t->min_tails[k] = INT32_MAX;
  t->min_tails[M - 1] = 0;
  for (int i = 0; i < N; i++) {
    tmp0 = p[(M - 1) * N + i];
    for (int k = M - 2; k >= 0; k--) {
      tmp1 = tmp0 + p[k * N + i];
      t->min_tails[k] = OR_MIN(t->min_tails[k], tmp0);
      tmp0 = tmp1;
    }
  }
}

/* lib/pfsp/Bound_johnson.chpl:50-87 (the LB2_LEARN branch is the one taken: all
 * i<j pairs in lexicographic order, identity machine_pair_order) */
static void fill_machine_pairs(or_pfsp_tables* t, int variant) {
  int c = 0;
  if (variant == 1) { /* LB2_NABESHIMA, :72-79: (i, i+1) */
    for (int i = 0; i < t->machines - 1; i++, c++) {
      t->mp0[c] = i;
      t->mp1[c] = i + 1;
      t->mp_order[c] = c;
    }
  } else if (variant == 2) { /* LB2_LAGEWEG, :80-87: (i, last) */
    for (int i = 0; i < t->machines - 1; i++, c++) {
      t->mp0[c] = i;
      t->mp1[c] = t->machines - 1;
      t->mp_order[c] = c;
    }
  } else { /* LB2_FULL / LB2_LEARN */
    for (int i = 0; i < t->machines - 1; i++)
      for (int j = i + 1; j < t->machines; j++) {
        t->mp0[c] = i;
        t->mp1[c] = j;
        t->mp_order[c] = c;
        c++;
      }
  }
  t->pairs = c; /* = machines*(machines-1)/2 resp. machines-1, Bound_johnson.chpl:36-43 */
}

/* lib/pfsp/Bound_johnson.chpl:89-104 — sum of p on the machines strictly between m1 and m2 */
static void fill_lags(or_pfsp_tables* t) {
  const int N = t->jobs;
  for (int i = 0; i < t->pairs; i++) {
    const int m1 = t->mp0[i], m2 = t->mp1[i];
    for (int j = 0; j < N; j++) {
      int32_t s = 0;
      for (int k = m1 + 1; k < m2; k++) s += t->p_times[k * N + j];
      t->lags[i * N + j] = s;
    }
  }
}

typedef struct {
  int32_t job, partition, ptm1, ptm2;
} johnson_job;

/* lib/pfsp/Bound_johnson.chpl:118-140 */
static int johnson_compare(const johnson_job* a, const johnson_job* b) {
  if (a->partition == 0 && b->partition == 1) return -1;
  if (a->partition == 1 && b->partition == 0) return 1;
  if (a->partition == 0) return a->ptm1 - b->ptm1;
  return b->ptm2 - a->ptm2;
}

/* lib/pfsp/Bound_johnson.chpl:145-177.  The sort is a stable insertion sort; tie order
 * may differ from Chapel's `sort` / libc qsort, which does not change any bound value
 * (Johnson's rule is tie-invariant; SURVEY §8c (iv)).  The table is an INPUT of the
 * GPU kernels, so kernel-vs-oracle parity is unaffected either way. */
static void fill_johnson_schedules(or_pfsp_tables* t) {
  const int N = t->jobs;
  johnson_job tmp[OR_MAX_JOBS];
  for (int k = 0; k < t->pairs; k++) {
    const int m1 = t->mp0[k], m2 = t->mp1[k];
    for (int i = 0; i < N; i++) {
      tmp[i].job = i;
      tmp[i].ptm1 = t->p_times[m1 * N + i] + t->lags[k * N + i];
      tmp[i].ptm2 = t->p_times[m2 * N + i] + t->lags[k * N + i];
      tmp[i].partition = (tmp[i].ptm1 < tmp[i].ptm2) ? 0 : 1;
    }
    for (int i = 1; i < N; i++) {
      johnson_job x = tmp[i];
      int j = i - 1;
      while (j >= 0 && johnson_compare(&tmp[j], &x) > 0) {
        tmp[j + 1] = tmp[j];
        j--;
      }
      tmp[j + 1] = x;
    }
    for (int i = 0; i < N; i++) t->johnson[k * N + i] = tmp[i].job;
  }
}

/* the fill_* precompute of pfsp_chpl.chpl:31-38 on any machine-major processing-time matrix p_times[k*jobs + j] */
int or_pfsp_tables_from_ptimes(or_pfsp_tables* t, int jobs, int machines, const int32_t* p_times, int heads_mode,
                               int variant) {
  if (jobs < 1 || jobs > OR_MAX_JOBS || machines < 1 || machines > OR_MAX_MACHINES) return -2;
  memset(t, 0, sizeof(*t));
  t->jobs = jobs;
  t->machines = machines;
  memcpy(t->p_times, p_times, (size_t)jobs * machines * sizeof(int32_t));
  fill_min_heads_tails(t, heads_mode);
  fill_machine_pairs(t, variant);
  fill_lags(t);
  fill_johnson_schedules(t);
  return 0;
}

/* pfsp_chpl.chpl:31-38 (module-scope table construction) */
int or_pfsp_tables_build_variant(or_pfsp_tables* t, int inst, int heads_mode, int variant) {
  if (inst < 1 || inst > 120) return -1;
  const int jobs = or_taillard_nb_jobs(inst), machines = or_taillard_nb_machines(inst);
  if (jobs > OR_MAX_JOBS) return -2; /* MAX_JOBS (20: only ta001..ta030, SURVEY A.2; 50: up to ta060) */
  int32_t p_times[OR_MAX_MACHINES * OR_MAX_JOBS];
  or_taillard_processing_times(p_times, inst);
  return or_pfsp_tables_from_ptimes(t, jobs, machines, p_times, heads_mode, variant);
}
int or_pfsp_tables_build(or_pfsp_tables* t, int inst, int heads_mode) {
  return or_pfsp_tables_build_variant(t, inst, heads_mode, 0);
}

/* ======================================================================== lb1 family */

/* lib/pfsp/Bound_simple.chpl:29-35 */
static void add_forward(int job, const or_pfsp_tables* t, int32_t* front) {
  const int N = t->jobs, M = t->machines;
  front[0] += t->p_times[job];
  for (int j = 1; j < M; j++) front[j] = OR_MAX(front[j - 1], front[j]) + t->p_times[j * N + job];
}

/* lib/pfsp/Bound_simple.chpl:47-62 */
static void schedule_front(const or_pfsp_tables* t, const int32_t* prmu, int limit1, int32_t* front) {
  if (limit1 == -1) {
    for (int i = 0; i < t->machines; i++) front[i] = t->min_heads[i];
    return;
  }
  for (int i = 0; i <= limit1; i++) add_forward(prmu[i], t, front);
}

/* lib/pfsp/Bound_simple.chpl:64-79; the general (limit2 < N) branch is kept for completeness */
static void schedule_back(const or_pfsp_tables* t, const int32_t* prmu, int limit2, int32_t* back) {
  const int N = t->jobs, M = t->machines;
  if (limit2 == N) {
    for (int i = 0; i < M; i++) back[i] = t->min_tails[i];
    return;
  }
  for (int k = N - 1; k >= limit2; k--) { /* Bound_simple.chpl:37-45 add_backward */
    const int job = prmu[k];
    back[M - 1] += t->p_times[(M - 1) * N + job];
    for (int j = M - 2; j >= 0; j--) back[j] = OR_MAX(back[j], back[j + 1]) + t->p_times[j * N + job];
  }
}

/* lib/pfsp/Bound_simple.chpl:94-106 */
static void sum_unscheduled(const or_pfsp_tables* t, const int32_t* prmu, int limit1, int limit2,
                            int32_t* remain) {
  const int N = t->jobs, M = t->machines;
  for (int k = limit1 + 1; k < limit2; k++) {
    const int job = prmu[k];
    for (int j = 0; j < M; j++) remain[j] += t->p_times[j * N + job];
  }
}

/* lib/pfsp/Bound_simple.chpl:108-121 */
static int32_t machine_bound_from_parts(const int32_t* front, const int32_t* back, const int32_t* remain,
                                        int nb_machines) {
  int32_t tmp0 = front[0] + remain[0];
  int32_t lb = tmp0 + back[0];
  for (int i = 1; i < nb_machines; i++) {
    int32_t tmp1 = OR_MAX(tmp0, front[i] + remain[i]);
    lb = OR_MAX(lb, tmp1 + back[i]);
    tmp0 = tmp1;
  }
  return lb;
}

/* lib/pfsp/Bound_simple.chpl:81-92 */
int32_t or_eval_solution(const or_pfsp_tables* t, const int32_t* prmu) {
  int32_t tmp[OR_MAX_MACHINES] = {0};
  for (int i = 0; i < t->jobs; i++) add_forward(prmu[i], t, tmp);
  return tmp[t->machines - 1];
}

/* lib/pfsp/Bound_simple.chpl:123-136.  Chapel zero-initialises three NUM_MACHINES(=20)
 * tuples and runs machine_bound_from_parts over all 20 entries (:135); the padding
 * entries are zero so the value equals the `machines`-long loop (SURVEY A.2) — we keep
 * the 20-long loop to follow the Chapel text. */
int32_t or_lb1_bound(const or_pfsp_tables* t, const int32_t* prmu, int32_t limit1, int32_t limit2) {
  int32_t front[OR_MAX_MACHINES] = {0}, back[OR_MAX_MACHINES] = {0}, remain[OR_MAX_MACHINES] = {0};
  schedule_front(t, prmu, limit1, front);
  schedule_back(t, prmu, limit2, back);
  sum_unscheduled(t, prmu, limit1, limit2, remain);
  return machine_bound_from_parts(front, back, remain, OR_MAX_MACHINES);
}

/* lib/pfsp/Bound_simple.chpl:197-222 */
static int32_t add_front_and_bound(const or_pfsp_tables* t, int job, const int32_t* front,
                                   const int32_t* back, const int32_t* remain) {
  const int N = t->jobs, M = t->machines;
  int32_t lb = front[0] + remain[0] + back[0];
  int32_t tmp0 = front[0] + t->p_times[job];
  for (int i = 1; i < M; i++) {
    int32_t tmp1 = OR_MAX(tmp0, front[i]);
    lb = OR_MAX(lb, tmp1 + remain[i] + back[i]);
    tmp0 = tmp1 + t->p_times[i * N + job];
  }
  return lb;
}

/* lib/pfsp/Bound_simple.chpl:138-161 (direction -1, the only live branch) */
void or_lb1_children_bounds(const or_pfsp_tables* t, const int32_t* prmu, int32_t limit1, int32_t limit2,
                            int32_t* lb_begin) {
  int32_t front[OR_MAX_MACHINES] = {0}, back[OR_MAX_MACHINES] = {0}, remain[OR_MAX_MACHINES] = {0};
  schedule_front(t, prmu, limit1, front);
  schedule_back(t, prmu, limit2, back);
  sum_unscheduled(t, prmu, limit1, limit2, remain);
  for (int i = 0; i < OR_MAX_JOBS; i++) lb_begin[i] = 0;
  for (int i = limit1 + 1; i < limit2; i++) {
    const int job = prmu[i];
    lb_begin[job] = add_front_and_bound(t, job, front, back, remain);
  }
}

/* ======================================================================== lb2 */

/* lib/pfsp/Bound_johnson.chpl:179-186 */
static void set_flags(const int32_t* prmu, int limit1, int limit2, int N, int32_t* flags) {
  for (int j = 0; j <= limit1; j++) flags[prmu[j]] = 1;
  for (int j = limit2; j < N; j++) flags[prmu[j]] = 1;
}

/* lib/pfsp/Bound_johnson.chpl:188-212 */
static int32_t compute_cmax_johnson(const or_pfsp_tables* t, const int32_t* flag, int32_t* tmp0,
                                    int32_t* tmp1, int ma0, int ma1, int ind) {
  const int N = t->jobs;
  for (int j = 0; j < N; j++) {
    const int job = t->johnson[ind * N + j];
    if (flag[job] == 0) {
      const int32_t ptm0 = t->p_times[ma0 * N + job];
      const int32_t ptm1 = t->p_times[ma1 * N + job];
      const int32_t lag = t->lags[ind * N + job];
      *tmp0 += ptm0;
      *tmp1 = OR_MAX(*tmp1, *tmp0 + lag);
      *tmp1 += ptm1;
    }
  }
  return *tmp1;
}

/* lib/pfsp/Bound_johnson.chpl:214-240 — note the early exit returns the running max at
 * the first pair (in machine_pair_order) where it exceeds minCmax (SURVEY A.5);
 * minCmax is a 64-bit Chapel int (max(int) under --ub 0). */
static int32_t lb_makespan(const or_pfsp_tables* t, const int32_t* flag, const int32_t* front,
                           const int32_t* back, int64_t minCmax) {
  int32_t lb = 0;
  for (int l = 0; l < t->pairs; l++) {
    const int i = t->mp_order[l];
    const int ma0 = t->mp0[i], ma1 = t->mp1[i];
    int32_t tmp0 = front[ma0], tmp1 = front[ma1];
    compute_cmax_johnson(t, flag, &tmp0, &tmp1, ma0, ma1, i);
    tmp1 = OR_MAX(tmp1 + back[ma1], tmp0 + back[ma0]);
    lb = OR_MAX(lb, tmp1);
    if ((int64_t)lb > minCmax) break;
  }
  return lb;
}

/* lib/pfsp/Bound_johnson.chpl:274-289 (set_flags is called with NUM_JOBS = 20, :286) */
int32_t or_lb2_bound(const or_pfsp_tables* t, const int32_t* prmu, int32_t limit1, int32_t limit2,
                     int64_t best) {
  int32_t front[OR_MAX_MACHINES] = {0}, back[OR_MAX_MACHINES] = {0};
  int32_t flags[OR_MAX_JOBS] = {0};
  schedule_front(t, prmu, limit1, front);
  schedule_back(t, prmu, limit2, back);
  set_flags(prmu, limit1, limit2, OR_MAX_JOBS, flags);
  return lb_makespan(t, flags, front, back, best);
}

/* ======================================================================== N-Queens */

/* nqueens_chpl.chpl:51-67 */
static uint8_t nq_is_safe(const uint8_t* board, int queen_num, int row_pos, int g) {
  uint8_t safe = 1;
  for (int i = 0; i < queen_num; i++) {
    const int other = board[i];
    for (int _g = 0; _g < g; _g++)
      if (other == row_pos - (queen_num - i) || other == row_pos + (queen_num - i)) safe = 0;
  }
  return safe;
}

/* nqueens_gpu_chpl.chpl:97-123 — one "thread" per (parent, k); only k >= depth is written */
void or_nq_evaluate_range(const or_nq_node* parents, int begin, int end, int N, int g, uint8_t* labels) {
  for (int pid = begin; pid < end; pid++) {
    const or_nq_node* parent = &parents[pid];
    const int depth = parent->depth;
    for (int k = 0; k < N; k++) {
      if (k >= depth) {
        const int queen_num = parent->board[k];
        uint8_t safe = 1;
        for (int i = 0; i < depth; i++) {
          const int pbi = parent->board[i];
          for (int _g = 0; _g < g; _g++)
            safe *= (uint8_t)(pbi != queen_num - (depth - i) && pbi != queen_num + (depth - i));
        }
        labels[(size_t)pid * N + k] = safe;
      }
    }
  }
}
void or_nq_evaluate(const or_nq_node* parents, int count, int N, int g, uint8_t* labels) {
  or_nq_evaluate_range(parents, 0, count, N, g, labels);
}

/* pfsp_gpu_chpl.chpl:192-208 (lb1), :216-235 (lb1_d), :238-254 (lb2), dispatch :257-270 */
void or_pfsp_evaluate_range(const or_pfsp_tables* t, int lb_kind, const or_pfsp_node* parents, int begin,
                            int end, int64_t best, int32_t* bounds) {
  const int jobs = t->jobs;
  for (int pid = begin; pid < end; pid++) {
    const or_pfsp_node* parent = &parents[pid];
    if (lb_kind == 0) {
      int32_t lb_begin[OR_MAX_JOBS];
      or_lb1_children_bounds(t, parent->prmu, parent->limit1, jobs, lb_begin);
      for (int k = 0; k < jobs; k++)
        if (k >= parent->limit1 + 1) bounds[(size_t)pid * jobs + k] = lb_begin[parent->prmu[k]];
    } else {
      int32_t prmu[OR_MAX_JOBS];
      memcpy(prmu, parent->prmu, sizeof(prmu));
      const int depth = parent->depth;
      for (int k = 0; k < jobs; k++) {
        if (k >= parent->limit1 + 1) {
          int32_t x = prmu[depth];
          prmu[depth] = prmu[k];
          prmu[k] = x;
          bounds[(size_t)pid * jobs + k] = (lb_kind == 1)
                                               ? or_lb1_bound(t, prmu, parent->limit1 + 1, jobs)
                                               : or_lb2_bound(t, prmu, parent->limit1 + 1, jobs, best);
          x = prmu[depth];
          prmu[depth] = prmu[k];
          prmu[k] = x;
        }
      }
    }
  }
}
void or_pfsp_evaluate(const or_pfsp_tables* t, int lb_kind, const or_pfsp_node* parents, int count,
                      int64_t best, int32_t* bounds) {
  or_pfsp_evaluate_range(t, lb_kind, parents, 0, count, best, bounds);
}

/* ======================================================================== pool (lib/commons/Pool.chpl) */

typedef struct {
  char* elements;
  size_t elt;
  int64_t capacity, front, size;
} or_pool;

static void pool_init(or_pool* p, size_t elt) { /* Pool.chpl:20-24, INITIAL_CAPACITY 1024 */
  p->elt = elt;
  p->capacity = 1024;
  p->front = 0;
  p->size = 0;
  p->elements = (char*)malloc((size_t)p->capacity * elt);
}
static void pool_free(or_pool* p) { free(p->elements); }
static void pool_push_back(or_pool* p, const void* node) { /* Pool.chpl:27-35 */
  if (p->front + p->size >= p->capacity) {
    p->capacity *= 2;
    p->elements = (char*)realloc(p->elements, (size_t)p->capacity * p->elt);
  }
  memcpy(p->elements + (size_t)(p->front + p->size) * p->elt, node, p->elt);
  p->size += 1;
}
static int pool_pop_back(or_pool* p, void* out) { /* Pool.chpl:38-47 */
  if (p->size > 0) {
    p->size -= 1;
    memcpy(out, p->elements + (size_t)(p->front + p->size) * p->elt, p->elt);
    return 1;
  }
  return 0;
}
static int pool_pop_front(or_pool* p, void* out) { /* Pool.chpl:62-73 */
  if (p->size > 0) {
    memcpy(out, p->elements + (size_t)p->front * p->elt, p->elt);
    p->front += 1;
    p->size -= 1;
    return 1;
  }
  return 0;
}
static int64_t pool_pop_back_bulk(or_pool* p, int64_t m, int64_t M, void* parents) { /* Pool.chpl:50-59 */
  if (p->size >= m) {
    const int64_t n = OR_MIN(p->size, M);
    p->size -= n;
    memcpy(parents, p->elements + (size_t)(p->front + p->size) * p->elt, (size_t)n * p->elt);
    return n;
  }
  return 0;
}

/* ======================================================================== N-Queens searches */

/* nqueens_chpl.chpl:70-89 */
static void nq_decompose(int N, int g, const or_nq_node* parent, uint64_t* tree, uint64_t* sol,
                         or_pool* pool) {
  const int depth = parent->depth;
  if (depth == N) {
    *sol += 1;
  } else {
    for (int j = depth; j < N; j++) {
      if (nq_is_safe(parent->board, depth, parent->board[j], g)) {
        or_nq_node child = *parent;
        child.depth = (uint8_t)(depth + 1);
        uint8_t x = child.board[depth];
        child.board[depth] = child.board[j];
        child.board[j] = x;
        pool_push_back(pool, &child);
        *tree += 1;
      }
    }
  }
}

static void nq_root(or_nq_node* root, int N) { /* NQueens_node.chpl:17-20 */
  memset(root, 0, sizeof(*root));
  for (int i = 0; i < N; i++) root->board[i] = (uint8_t)i;
}

/* nqueens_chpl.chpl:92-113 */
void or_nq_search_seq(int N, int g, or_search_result* r) {
  memset(r, 0, sizeof(*r));
  or_pool pool;
  pool_init(&pool, sizeof(or_nq_node));
  or_nq_node root, parent;
  nq_root(&root, N);
  pool_push_back(&pool, &root);
  const double t0 = now_s();
  while (pool_pop_back(&pool, &parent)) nq_decompose(N, g, &parent, &r->tree, &r->sol, &pool);
  r->seconds = now_s() - t0;
  pool_free(&pool);
}

/* the same sequential search started from given nodes (bench.py's CPU legs: one share of the tree per host
 * thread), and the breadth-first frontier of depth `depth` it is started from; nqueens_chpl.chpl:92-113 */
void or_nq_search_from(int N, int g, const or_nq_node* nodes, int n, uint64_t* tree, uint64_t* sol) {
  or_pool pool;
  pool_init(&pool, sizeof(or_nq_node));
  or_nq_node parent;
  for (int i = 0; i < n; i++) pool_push_back(&pool, &nodes[i]);
  while (pool_pop_back(&pool, &parent)) nq_decompose(N, g, &parent, tree, sol, &pool);
  pool_free(&pool);
}
int or_nq_frontier(int N, int g, int depth, or_nq_node* out, int cap, uint64_t* tree, uint64_t* sol) {
  or_pool pool;
  pool_init(&pool, sizeof(or_nq_node));
  or_nq_node root, parent;
  nq_root(&root, N);
  pool_push_back(&pool, &root);
  int n = 0;
  while (pool_pop_front(&pool, &parent)) {
    if (parent.depth >= depth) {
      if (n >= cap) {
        pool_free(&pool);
        return -1;
      }
      out[n++] = parent;
    } else {
      nq_decompose(N, g, &parent, tree, sol, &pool);
    }
  }
  pool_free(&pool);
  return n;
}

/* nqueens_gpu_chpl.chpl:126-149 */
static void nq_generate_children(int N, const or_nq_node* parents, int64_t size, const uint8_t* labels,
                                 uint64_t* tree, uint64_t* sol, or_pool* pool) {
  for (int64_t i = 0; i < size; i++) {
    const or_nq_node* parent = &parents[i];
    const int depth = parent->depth;
    if (depth == N) {
      *sol += 1;
    } else {
      for (int j = depth; j < N; j++) {
        if (labels[j + i * N] == 1) {
          or_nq_node child = *parent;
          child.depth = (uint8_t)(depth + 1);
          uint8_t x = child.board[depth];
          child.board[depth] = child.board[j];
          child.board[j] = x;
          pool_push_back(pool, &child);
          *tree += 1;
        }
      }
    }
  }
}

/* evaluate_gpu + generate_children of one chunk (nqueens_gpu_chpl.chpl:97-149): the children, in the
 * reference's order, as they would be appended to the pool */
int64_t or_nq_expand_chunk(const or_nq_node* parents, int count, int N, int g, or_nq_node* children,
                           int64_t capacity, uint64_t* solutions) {
  uint8_t* labels = (uint8_t*)malloc((size_t)count * N + 1);
  or_pool pool;
  pool_init(&pool, sizeof(or_nq_node));
  uint64_t tree = 0, sol = 0;
  memset(labels, 0xCD, (size_t)count * N + 1);
  or_nq_evaluate(parents, count, N, g, labels);
  nq_generate_children(N, parents, count, labels, &tree, &sol, &pool);
  const int64_t n = pool.size;
  if (n <= capacity) memcpy(children, pool.elements + (size_t)pool.front * pool.elt, (size_t)n * sizeof(or_nq_node));
  if (solutions) *solutions = sol;
  pool_free(&pool);
  free(labels);
  return n;
}

/* offload loop of one pool: nqueens_gpu_chpl.chpl:197-215; capture hook for tests */
typedef struct {
  int which;
  void* out;
  int cap, got;
  int64_t best_at_launch;
  int64_t counter;
} capture_t;

static void nq_offload_loop(int N, int g, int m, int M, or_pool* pool, or_search_result* r,
                            or_nq_node* parents, uint8_t* labels, capture_t* cap) {
  for (;;) {
    const int64_t n = pool_pop_back_bulk(pool, m, M, parents);
    if (n <= 0) break;
    if (cap && cap->counter++ == cap->which) {
      cap->got = (int)OR_MIN(n, (int64_t)cap->cap);
      memcpy(cap->out, parents, (size_t)cap->got * sizeof(or_nq_node));
    }
    memset(labels, 0xCD, (size_t)n * N); /* the reference leaves stale garbage below the live range */
    or_nq_evaluate(parents, (int)n, N, g, labels);
    r->offloads += 1;
    r->offloaded_parents += (uint64_t)n;
    for (int64_t i = 0; i < n; i++) {
      r->depth_hist[parents[i].depth] += 1;
      r->live_slots += (uint64_t)(N - parents[i].depth);
    }
    nq_generate_children(N, parents, n, labels, &r->tree, &r->sol, pool);
  }
}

/* step-2 counts of task `gpu`: what the task added to r since `tree0` / `sol0` */
static void note_task(or_search_result* r, int gpu, uint64_t tree0, uint64_t sol0, int64_t best) {
  if (gpu < 0 || gpu >= 8) return;
  r->task_tree[gpu] = r->tree - tree0;
  r->task_sol[gpu] = r->sol - sol0;
  r->task_best[gpu] = best;
}

/* nqueens_gpu_chpl.chpl:152-248 (D == 1) and nqueens_multigpu_chpl.chpl:158-352 (D > 1,
 * static strided split :199-226, no work stealing — counts are split-invariant).  part >= 0: that task alone
 * (or_nq_search_offload_part); warm: the step-1 pool size */
static void nq_search_offload_impl(int N, int g, int m, int M, int D, int part, int64_t warm, or_search_result* r,
                                   capture_t* cap) {
  memset(r, 0, sizeof(*r));
  or_pool pool;
  pool_init(&pool, sizeof(or_nq_node));
  or_nq_node root, parent;
  nq_root(&root, N);
  pool_push_back(&pool, &root);
  or_nq_node* parents = (or_nq_node*)malloc((size_t)M * sizeof(or_nq_node));
  uint8_t* labels = (uint8_t*)malloc((size_t)M * N);
  const double t0 = now_s();

  /* step 1 */
  while (pool.size < warm) {
    if (!pool_pop_front(&pool, &parent)) break;
    nq_decompose(N, g, &parent, &r->tree, &r->sol, &pool);
  }
  if (part > 0) r->tree = r->sol = 0; /* step 1 is credited to part 0 */
  /* step 2 */
  if (D <= 1) {
    const uint64_t tree0 = r->tree, sol0 = r->sol;
    nq_offload_loop(N, g, m, M, &pool, r, parents, labels, cap);
    note_task(r, 0, tree0, sol0, 0);
  } else {
    const int64_t poolSize = pool.size, c = poolSize / D, l = poolSize - (int64_t)(D - 1) * c, f = pool.front;
    pool.front = 0;
    pool.size = 0;
    or_pool* multi = (or_pool*)malloc((size_t)D * sizeof(or_pool));
    for (int gpu = 0; gpu < D; gpu++) {
      pool_init(&multi[gpu], sizeof(or_nq_node));
      for (int64_t i = 0; i < c; i++)
        pool_push_back(&multi[gpu], pool.elements + (size_t)(gpu + f + i * D) * pool.elt);
      if (gpu == D - 1)
        for (int64_t i = 0; i < l - c; i++)
          pool_push_back(&multi[gpu], pool.elements + (size_t)(D * c + f + i) * pool.elt);
    }
    for (int gpu = 0; gpu < D; gpu++) {
      if (part < 0 || gpu == part) { /* a part leaves the other tasks' nodes to the other parts */
        const uint64_t tree0 = r->tree, sol0 = r->sol;
        nq_offload_loop(N, g, m, M, &multi[gpu], r, parents, labels, NULL);
        note_task(r, gpu, tree0, sol0, 0);
        while (pool_pop_back(&multi[gpu], &parent)) pool_push_back(&pool, &parent); /* :315-320 */
      }
      pool_free(&multi[gpu]);
    }
    free(multi);
  }
  /* step 3 */
  while (pool_pop_back(&pool, &parent)) nq_decompose(N, g, &parent, &r->tree, &r->sol, &pool);
  r->seconds = now_s() - t0;
  free(parents);
  free(labels);
  pool_free(&pool);
}

void or_nq_search_offload(int N, int g, int m, int M, int D, or_search_result* r) {
  nq_search_offload_impl(N, g, m, M, D, -1, (int64_t)D * m, r, NULL);
}

void or_nq_search_offload_part(int N, int g, int m, int M, int D, int part, int warm, or_search_result* r) {
  nq_search_offload_impl(N, g, m, M, D, part, warm, r, NULL);
}

int or_nq_capture_chunk(int N, int g, int m, int M, int which, or_nq_node* out, int cap) {
  capture_t c = {which, out, cap, -1, 0, 0};
  or_search_result r;
  nq_search_offload_impl(N, g, m, M, 1, -1, m, &r, &c);
  return c.got;
}

/* ======================================================================== PFSP searches */

static void pfsp_root(or_pfsp_node* root, int jobs) { /* PFSP_node.chpl:18-23 */
  memset(root, 0, sizeof(*root));
  root->limit1 = -1;
  for (int i = 0; i < jobs; i++) root->prmu[i] = i;
}

static void pfsp_make_child(const or_pfsp_node* parent, int i, or_pfsp_node* child) {
  *child = *parent;
  child->depth = parent->depth + 1;
  child->limit1 = parent->limit1 + 1;
  int32_t x = child->prmu[parent->depth];
  child->prmu[parent->depth] = child->prmu[i];
  child->prmu[i] = x;
}

/* pfsp_chpl.chpl:88-189: decompose_lb1 :88-113, decompose_lb1_d :115-145, decompose_lb2 :147-172.
 * `best` is updated between siblings on this sequential path. */
static void pfsp_decompose(const or_pfsp_tables* t, int lb_kind, const or_pfsp_node* parent, uint64_t* tree,
                           uint64_t* sol, int64_t* best, or_pool* pool) {
  const int jobs = t->jobs;
  int32_t lb_begin[OR_MAX_JOBS];
  if (lb_kind == 0) or_lb1_children_bounds(t, parent->prmu, parent->limit1, jobs, lb_begin);
  for (int i = parent->limit1 + 1; i < jobs; i++) {
    or_pfsp_node child;
    pfsp_make_child(parent, i, &child);
    int32_t lowerbound;
    if (lb_kind == 0)
      lowerbound = lb_begin[parent->prmu[i]];
    else if (lb_kind == 1)
      lowerbound = or_lb1_bound(t, child.prmu, child.limit1, jobs);
    else
      lowerbound = or_lb2_bound(t, child.prmu, child.limit1, jobs, *best);
    if (child.depth == jobs) {
      *sol += 1;
      if (lowerbound < *best) *best = lowerbound;
    } else if (lowerbound < *best) {
      pool_push_back(pool, &child);
      *tree += 1;
    }
  }
}

/* pfsp_chpl.chpl:191-215 */
void or_pfsp_search_seq(int inst, int lb_kind, int ub, int heads_mode, or_search_result* r) {
  memset(r, 0, sizeof(*r));
  or_pfsp_tables* t = (or_pfsp_tables*)malloc(sizeof(*t));
  if (or_pfsp_tables_build(t, inst, heads_mode) != 0) {
    free(t);
    r->best = -1;
    return;
  }
  int64_t best = (ub == 1) ? or_taillard_best_ub(inst) : INT64_MAX; /* pfsp_chpl.chpl:29 */
  or_pool pool;
  pool_init(&pool, sizeof(or_pfsp_node));
  or_pfsp_node root, parent;
  pfsp_root(&root, t->jobs);
  pool_push_back(&pool, &root);
  const double t0 = now_s();
  while (pool_pop_back(&pool, &parent)) pfsp_decompose(t, lb_kind, &parent, &r->tree, &r->sol, &best, &pool);
  r->seconds = now_s() - t0;
  r->best = best;
  pool_free(&pool);
  free(t);
}

/* pfsp_gpu_chpl.chpl:273-303 */
static void pfsp_generate_children(int jobs, const or_pfsp_node* parents, int64_t size, const int32_t* bounds,
                                   uint64_t* tree, uint64_t* sol, int64_t* best, or_pool* pool) {
  for (int64_t i = 0; i < size; i++) {
    const or_pfsp_node* parent = &parents[i];
    const int depth = parent->depth;
    for (int j = parent->limit1 + 1; j < jobs; j++) {
      const int32_t lowerbound = bounds[j + i * jobs];
      if (depth + 1 == jobs) {
        *sol += 1;
        if (lowerbound < *best) *best = lowerbound;
      } else if (lowerbound < *best) {
        or_pfsp_node child;
        pfsp_make_child(parent, j, &child);
        pool_push_back(pool, &child);
        *tree += 1;
      }
    }
  }
}

/* evaluate_gpu + generate_children of one PFSP chunk (pfsp_gpu_chpl.chpl:384-392): bounds with `best` at
 * launch, then the sequential rule of generate_children (best lowered by leaves while the chunk is walked) */
int64_t or_pfsp_expand_chunk(const or_pfsp_tables* t, int lb_kind, const or_pfsp_node* parents, int count,
                             int64_t* best, or_pfsp_node* children, int64_t capacity, uint64_t* solutions) {
  const int jobs = t->jobs;
  int32_t* bounds = (int32_t*)malloc(((size_t)count * jobs + 1) * sizeof(int32_t));
  or_pool pool;
  pool_init(&pool, sizeof(or_pfsp_node));
  uint64_t tree = 0, sol = 0;
  memset(bounds, 0xCD, ((size_t)count * jobs + 1) * sizeof(int32_t));
  or_pfsp_evaluate(t, lb_kind, parents, count, *best, bounds);
  pfsp_generate_children(jobs, parents, count, bounds, &tree, &sol, best, &pool);
  const int64_t n = pool.size;
  if (n <= capacity && n > 0)
    memcpy(children, pool.elements + (size_t)pool.front * pool.elt, (size_t)n * sizeof(or_pfsp_node));
  if (solutions) *solutions = sol;
  pool_free(&pool);
  free(bounds);
  return n;
}

/* pfsp_gpu_chpl.chpl:373-396: `best` is the value AT LAUNCH for the whole chunk */
static void pfsp_offload_loop(const or_pfsp_tables* t, int lb_kind, int m, int M, or_pool* pool, int64_t* best,
                              or_search_result* r, or_pfsp_node* parents, int32_t* bounds, capture_t* cap) {
  const int jobs = t->jobs;
  for (;;) {
    const int64_t n = pool_pop_back_bulk(pool, m, M, parents);
    if (n <= 0) break;
    if (cap && cap->counter++ == cap->which) {
      cap->got = (int)OR_MIN(n, (int64_t)cap->cap);
      cap->best_at_launch = *best;
      memcpy(cap->out, parents, (size_t)cap->got * sizeof(or_pfsp_node));
    }
    memset(bounds, 0xCD, (size_t)n * jobs * sizeof(int32_t));
    or_pfsp_evaluate(t, lb_kind, parents, (int)n, *best, bounds);
    r->offloads += 1;
    r->offloaded_parents += (uint64_t)n;
    for (int64_t i = 0; i < n; i++) {
      r->depth_hist[parents[i].depth] += 1;
      r->live_slots += (uint64_t)(jobs - parents[i].limit1 - 1);
    }
    pfsp_generate_children(jobs, parents, n, bounds, &r->tree, &r->sol, best, pool);
  }
}

/* pfsp_gpu_chpl.chpl:306-431 (D == 1); pfsp_multigpu_chpl.chpl:316-560 (D > 1: per-task best_l
 * starting from `best` :384, `min reduce` at the end :520, static split, no stealing).  part >= 0: that task
 * alone (or_pfsp_search_offload_part), whose step 3 then runs with its own best_l */
static void pfsp_search_offload_impl(int inst, int lb_kind, int ub, int m, int M, int D, int part, int heads_mode,
                                     or_search_result* r, capture_t* cap) {
  memset(r, 0, sizeof(*r));
  or_pfsp_tables* t = (or_pfsp_tables*)malloc(sizeof(*t));
  if (or_pfsp_tables_build(t, inst, heads_mode) != 0) {
    free(t);
    r->best = -1;
    return;
  }
  const int jobs = t->jobs;
  int64_t best = (ub == 1) ? or_taillard_best_ub(inst) : INT64_MAX;
  or_pool pool;
  pool_init(&pool, sizeof(or_pfsp_node));
  or_pfsp_node root, parent;
  pfsp_root(&root, jobs);
  pool_push_back(&pool, &root);
  or_pfsp_node* parents = (or_pfsp_node*)malloc((size_t)M * sizeof(or_pfsp_node));
  int32_t* bounds = (int32_t*)malloc((size_t)M * jobs * sizeof(int32_t));
  const double t0 = now_s();

  while (pool.size < (int64_t)D * m) {
    if (!pool_pop_front(&pool, &parent)) break;
    pfsp_decompose(t, lb_kind, &parent, &r->tree, &r->sol, &best, &pool);
  }
  if (part > 0) r->tree = r->sol = 0; /* step 1 is credited to part 0 */
  if (D <= 1) {
    const uint64_t tree0 = r->tree, sol0 = r->sol;
    pfsp_offload_loop(t, lb_kind, m, M, &pool, &best, r, parents, bounds, cap);
    note_task(r, 0, tree0, sol0, best);
  } else {
    const int64_t poolSize = pool.size, c = poolSize / D, l = poolSize - (int64_t)(D - 1) * c, f = pool.front;
    pool.front = 0;
    pool.size = 0;
    int64_t best_min = best;
    or_pool* multi = (or_pool*)malloc((size_t)D * sizeof(or_pool));
    for (int gpu = 0; gpu < D; gpu++) { /* every task takes its chunk first (:386-398) */
      pool_init(&multi[gpu], sizeof(or_pfsp_node));
      for (int64_t i = 0; i < c; i++)
        pool_push_back(&multi[gpu], pool.elements + (size_t)(gpu + f + i * D) * pool.elt);
      if (gpu == D - 1)
        for (int64_t i = 0; i < l - c; i++)
          pool_push_back(&multi[gpu], pool.elements + (size_t)(D * c + f + i) * pool.elt);
    }
    for (int gpu = 0; gpu < D; gpu++) {
      if (part < 0 || gpu == part) { /* a part leaves the other tasks' nodes to the other parts */
        int64_t best_l = best;
        const uint64_t tree0 = r->tree, sol0 = r->sol;
        pfsp_offload_loop(t, lb_kind, m, M, &multi[gpu], &best_l, r, parents, bounds, NULL);
        note_task(r, gpu, tree0, sol0, best_l);
        best_min = OR_MIN(best_min, best_l);
        while (pool_pop_back(&multi[gpu], &parent)) pool_push_back(&pool, &parent);
      }
      pool_free(&multi[gpu]);
    }
    free(multi);
    best = best_min;
  }
  while (pool_pop_back(&pool, &parent)) pfsp_decompose(t, lb_kind, &parent, &r->tree, &r->sol, &best, &pool);
  r->seconds = now_s() - t0;
  r->best = best;
  free(parents);
  free(bounds);
  pool_free(&pool);
  free(t);
}

void or_pfsp_search_offload(int inst, int lb_kind, int ub, int m, int M, int D, int heads_mode,
                            or_search_result* r) {
  pfsp_search_offload_impl(inst, lb_kind, ub, m, M, D, -1, heads_mode, r, NULL);
}

void or_pfsp_search_offload_part(int inst, int lb_kind, int ub, int m, int M, int D, int part, int heads_mode,
                                 or_search_result* r) {
  pfsp_search_offload_impl(inst, lb_kind, ub, m, M, D, part, heads_mode, r, NULL);
}

int or_pfsp_capture_chunk(int inst, int lb_kind, int ub, int m, int M, int which, or_pfsp_node* out, int cap,
                          int64_t* best_at_launch) {
  capture_t c = {which, out, cap, -1, 0, 0};
  or_search_result r;
  pfsp_search_offload_impl(inst, lb_kind, ub, m, M, 1, -1, 0, &r, &c);
  if (best_at_launch) *best_at_launch = c.best_at_launch;
  return c.got;
}

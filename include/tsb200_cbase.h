/*
 * tsb200_cbase.h — C ABI of libtsb200_cbase.so, a link-level drop-in for the GPU offload step of the reference's
 * C+CUDA PFSP drivers (baselines/pfsp/pfsp_gpu_cuda.c, pfsp_multigpu_cuda.c).
 *
 * Those drivers reach the GPU through one function, evaluate_gpu (baselines/pfsp/lib/evaluate.h:12-13, defined in
 * lib/evaluate.cu).  This library exports a function of that name, signature and C linkage, so that a driver linked
 * with -ltsb200_cbase in place of evaluate.o runs the sm_90a kernels of libtsb200.so (tsb_pfsp_evaluate_device)
 * with no source change.  Its own pool, popBackBulk, generate_children, cudaMemcpys, multi-GPU split and work
 * stealing are untouched.
 *
 * The three records below restate the reference's definitions (baselines/pfsp/lib/PFSP_node.h,
 * c_bound_simple.h, c_bound_johnson.h) field for field, for a build with MAX_JOBS = 20: the structs are passed by
 * value, so their layout is part of the ABI.
 *
 * evaluate_gpu(jobs, lb, size, nbBlocks, best, lbound1, lbound2, parents, bounds):
 *   lb        0 = lb1_d, 1 = lb1, 2 = lb2 (TSB_LB1_D, TSB_LB1, TSB_LB2 of tsb200.h)
 *   size      jobs * poolSize; bounds[p*jobs + k] is written for k >= parents[p].limit1 + 1
 *   nbBlocks  ignored (the kernels choose their own grids)
 *   best      read once, at the call, for lb2's early exit (as evaluate.cu:111 does); never written
 *   lbound1/2 the caller's DEVICE tables (structs of device pointers), as the drivers build them
 *   parents, bounds  device pointers on the calling thread's current device
 * The kernel runs on the legacy default stream, as the reference's launch does, so that the caller's following
 * plain cudaMemcpy of `bounds` waits for it.
 *
 * Tables: the first call that sees a given key — calling thread, current device, the eight table pointers and
 * nb_jobs / nb_machines / nb_machine_pairs — copies the tables to the host and builds a libtsb200 handle from them
 * (tsb_pfsp_create: the library's own packing, validation and kernel route).  That handle serves every later call
 * with the same key.  The library ASSUMES that the tables behind a key never change after that first call: the
 * reference builds them once before its search and frees them after it.  A program that rewrites its tables in place
 * must call tsb_cbase_release() first.  Chunks larger than the first call's are fine: tsb_pfsp_evaluate_device is not
 * bounded by a handle's M_max.  Thread-safe: D threads of pfsp_multigpu_cuda, each with its own tables on its own
 * GPU, call it at once.
 *
 * Refusals and failures: evaluate_gpu returns void, so a call it cannot serve writes one line to stderr, with
 * tsb_strerror and tsb_last_cuda_error, and leaves `bounds` unwritten.  It cannot serve: jobs other than 20 (the
 * build's MAX_JOBS; tsb_pfsp_create takes 20-job instances only, ta001..ta030), lb outside 0..2, size not a multiple
 * of jobs, a null pointer, tables tsb_pfsp_create refuses, lb2 on tables whose handle refuses lb2 (tsb200.h), a
 * failing CUDA call.  The first such code sticks: tsb_cbase_status() returns it until tsb_cbase_release().  The
 * library never calls exit() or abort().
 */
#ifndef TSB200_CBASE_H
#define TSB200_CBASE_H

#ifdef __cplusplus
extern "C" {
#endif

/* baselines/pfsp/lib/PFSP_node.h (MAX_JOBS 20): 88 bytes */
typedef struct {
  int depth;
  int limit1;
  int prmu[20];
} Node;

/* baselines/pfsp/lib/c_bound_simple.h: 32 bytes on LP64 */
struct lb1_bound_data {
  int* p_times;   /* [nb_machines * nb_jobs], machine-major */
  int* min_heads; /* [nb_machines] */
  int* min_tails; /* [nb_machines] */
  int nb_jobs;
  int nb_machines;
};
typedef struct lb1_bound_data lb1_bound_data;

/* baselines/pfsp/lib/c_bound_johnson.h: 56 bytes on LP64 */
typedef struct lb2_bound_data {
  int* johnson_schedules;  /* [nb_machine_pairs * nb_jobs] */
  int* lags;               /* [nb_machine_pairs * nb_jobs] */
  int* machine_pairs_1;    /* [nb_machine_pairs] */
  int* machine_pairs_2;    /* [nb_machine_pairs] */
  int* machine_pair_order; /* [nb_machine_pairs] */
  int nb_machine_pairs;
  int nb_jobs;
  int nb_machines;
} lb2_bound_data;

void evaluate_gpu(const int jobs, const int lb, const int size, const int nbBlocks, int* best,
                  const lb1_bound_data lbound1, const lb2_bound_data lbound2, Node* parents, int* bounds);

/* TSB_OK (0), or the first TSB_E* code (tsb200.h) a call of evaluate_gpu met since load or the last release */
int tsb_cbase_status(void);
/* destroys every cached handle and clears the status; call it while no evaluate_gpu is running */
void tsb_cbase_release(void);

#ifdef __cplusplus
}
#endif

#endif /* TSB200_CBASE_H */

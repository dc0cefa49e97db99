/* sizeof and offsetof of the three records the reference's evaluate_gpu takes (Node, lb1_bound_data,
 * lb2_bound_data), one "record field offset" line each plus one "record sizeof size" line.  Built twice: against the
 * reference's own headers by oracle/cbase.mk (-> _ref/cbase_layout.txt), and against include/tsb200_cbase.h with
 * -DTSB_CBASE by tests/test_cbase.py; the two outputs must be equal. */
#include <stddef.h>
#include <stdio.h>

#ifdef TSB_CBASE
#include "tsb200_cbase.h"
#else
#include "PFSP_node.h"
#include "c_bound_johnson.h"
#include "c_bound_simple.h"
#endif

#define SIZE(T) printf(#T " sizeof %zu\n", sizeof(T))
#define OFF(T, f) printf(#T " " #f " %zu\n", offsetof(T, f))

int main(void) {
  SIZE(Node);
  OFF(Node, depth);
  OFF(Node, limit1);
  OFF(Node, prmu);
  SIZE(lb1_bound_data);
  OFF(lb1_bound_data, p_times);
  OFF(lb1_bound_data, min_heads);
  OFF(lb1_bound_data, min_tails);
  OFF(lb1_bound_data, nb_jobs);
  OFF(lb1_bound_data, nb_machines);
  SIZE(lb2_bound_data);
  OFF(lb2_bound_data, johnson_schedules);
  OFF(lb2_bound_data, lags);
  OFF(lb2_bound_data, machine_pairs_1);
  OFF(lb2_bound_data, machine_pairs_2);
  OFF(lb2_bound_data, machine_pair_order);
  OFF(lb2_bound_data, nb_machine_pairs);
  OFF(lb2_bound_data, nb_jobs);
  OFF(lb2_bound_data, nb_machines);
  return 0;
}

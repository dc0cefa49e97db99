"""tsb200 — Python host-side mirror of the reference's GPU offload interface, on top of the C ABI
(include/tsb200.h) of the H100-native evaluator library libtsb200.so.

The reference's Chapel drivers call, per offload round (nqueens_gpu_chpl.chpl:203-205,
pfsp_gpu_chpl.chpl:384-386):

    parents_d = parents;  on device do evaluate_gpu(parents_d, size, ...);  labels = labels_d;

`NQueensEvaluator.evaluate_gpu` / `PfspEvaluator.evaluate_gpu` are that step with the same argument
meaning (`size` = N*poolSize resp. jobs*poolSize, results in `labels` / `bounds`), numpy structured
arrays standing for the Chapel records.  There is no CPU fallback: without libtsb200.so or a CUDA
device every call raises.
"""
from ._lib import (LB1, LB1_D, LB2, ROUTE_LB2, ROUTE_LB2U, ROUTE_MT_MASK, ROUTE_SIMD16, XFER_AUTO, XFER_MEMCPY,
                   XFER_ZEROCOPY, PfspTables, PfspTables50, SearchStats, TsbError, check, lib)
from .nqueens import (NQ_NODE_DTYPE, NQueensEvaluator, nqueens_search, nqueens_search_device,
                      nqueens_pool_run_multi, nqueens_search_device_part, nqueens_warmup)
from .pfsp import (PFSP_NODE_DTYPE, PFSP_NODE50_DTYPE, LB_NAMES, LB2_VARIANTS, PfspEvaluator, taillard_tables50, pfsp_search, pfsp_search_device,
                   pfsp_search_device_part, taillard_tables)

__all__ = ["NQueensEvaluator", "PfspEvaluator", "nqueens_warmup", "nqueens_pool_run_multi", "nqueens_search", "nqueens_search_device", "nqueens_search_device_part", "pfsp_search", "pfsp_search_device",
           "pfsp_search_device_part",
           "taillard_tables",
           "NQ_NODE_DTYPE", "PFSP_NODE_DTYPE", "PFSP_NODE50_DTYPE", "LB2_VARIANTS", "taillard_tables50", "LB_NAMES", "LB1", "LB1_D", "LB2", "TsbError", "lib", "check",
           "PfspTables", "PfspTables50", "SearchStats", "XFER_AUTO", "XFER_MEMCPY", "XFER_ZEROCOPY",
           "ROUTE_MT_MASK", "ROUTE_SIMD16", "ROUTE_LB2", "ROUTE_LB2U"]

# oracle/cbase.mk — the reference's C+CUDA PFSP drivers, built twice: as the reference builds them (with its own
# lib/evaluate.cu, by nvcc for sm_90a) and relinked against libtsb200_cbase.so in place of evaluate.o.
# TEST INFRASTRUCTURE, like everything under oracle/ (tests/test_cbase.py, tests/test_gpu_cbase.py, tools/cbase_time.py).
#
#   make -f cbase.mk     -> _ref/pfsp_gpu_cuda.out       _ref/pfsp_multigpu_cuda.out      (unmodified)
#                           _ref/pfsp_gpu_cuda_tsb.out   _ref/pfsp_multigpu_cuda_tsb.out  (same objects, -ltsb200_cbase)
#                           _ref/cbase_layout.txt        (sizeof / offsetof of the records evaluate_gpu takes)
#
# The reference's sources are compiled where they lie under $(REF); objects go to _ref/cbase/ (git-ignored).  Its
# makefile is not run: it targets sm_86 and a cluster's include paths.  Its .c drivers include <cuda.h> but call the
# runtime API, so gcc gets -include cuda_runtime.h.  The MPI driver (pfsp_dist_multigpu_cuda.c) needs mpicc and is
# not built.  The _tsb binaries find libtsb200_cbase.so through an rpath relative to themselves, so the tree can move.
TSB200_REFERENCE ?= $(abspath $(CURDIR)/../../reference)
REF  ?= $(TSB200_REFERENCE)
CC   ?= gcc
NVCC ?= nvcc
CUDA ?= /usr/local/cuda

PF  := $(REF)/baselines/pfsp
COM := $(REF)/baselines/commons
PKG := ../gpu-accelerated-tree-search-chapel_b200
O   := _ref/cbase

CFLAGS_C := -O3 -w -I$(CUDA)/include -include cuda_runtime.h
LDCUDA   := -lm -L$(CUDA)/lib64 -lcudart -Wl,-rpath,$(CUDA)/lib64
# (what -fopenmp adds at link time, spelled out: a gcc without its libgomp.spec and libgomp.so link names still finds
# the runtime library itself)
LDOMP    := -l:libgomp.so.1 -lpthread
LDTSB    := -L$(PKG) -ltsb200_cbase -Wl,-rpath,'$$ORIGIN/../$(PKG)'

LIB_OBJ := $(O)/c_taillard.o $(O)/c_bound_simple.o $(O)/c_bound_johnson.o $(O)/PFSP_node.o
GPU_OBJ := $(O)/pfsp_gpu_cuda.o $(LIB_OBJ) $(O)/Pool.o
MGPU_OBJ := $(O)/pfsp_multigpu_cuda.o $(LIB_OBJ) $(O)/Pool_ext.o $(O)/util.o

all: _ref/pfsp_gpu_cuda.out _ref/pfsp_multigpu_cuda.out _ref/pfsp_gpu_cuda_tsb.out _ref/pfsp_multigpu_cuda_tsb.out \
     _ref/cbase_layout.txt

$(O)/.dir:
	mkdir -p $(O)
	touch $@

$(O)/%.o: $(PF)/lib/%.c $(O)/.dir
	$(CC) $(CFLAGS_C) -c $< -o $@
$(O)/util.o: $(COM)/util.c $(O)/.dir
	$(CC) $(CFLAGS_C) -c $< -o $@
$(O)/pfsp_gpu_cuda.o: $(PF)/pfsp_gpu_cuda.c $(O)/.dir
	$(CC) $(CFLAGS_C) -c $< -o $@
$(O)/pfsp_multigpu_cuda.o: $(PF)/pfsp_multigpu_cuda.c $(O)/.dir
	$(CC) $(CFLAGS_C) -fopenmp -c $< -o $@
# the reference's own kernels (evaluate.cu #includes c_bounds_gpu.cu from its directory)
$(O)/evaluate.o: $(PF)/lib/evaluate.cu $(O)/.dir
	$(NVCC) -O3 -gencode arch=compute_90a,code=sm_90a -w -c $< -o $@

_ref/pfsp_gpu_cuda.out: $(GPU_OBJ) $(O)/evaluate.o
	$(CC) -o $@ $^ $(LDCUDA)
_ref/pfsp_multigpu_cuda.out: $(MGPU_OBJ) $(O)/evaluate.o
	$(CC) -o $@ $^ $(LDOMP) $(LDCUDA)
_ref/pfsp_gpu_cuda_tsb.out: $(GPU_OBJ) $(PKG)/libtsb200_cbase.so
	$(CC) -o $@ $(GPU_OBJ) $(LDTSB) $(LDCUDA)
_ref/pfsp_multigpu_cuda_tsb.out: $(MGPU_OBJ) $(PKG)/libtsb200_cbase.so
	$(CC) -o $@ $(MGPU_OBJ) $(LDTSB) $(LDOMP) $(LDCUDA)

_ref/cbase_layout.txt: cbase_layout.c $(O)/.dir
	$(CC) -O2 -Wall -I$(PF)/lib -o $(O)/cbase_layout cbase_layout.c
	$(O)/cbase_layout > $@

clean:
	rm -rf $(O) _ref/pfsp_gpu_cuda.out _ref/pfsp_multigpu_cuda.out _ref/pfsp_gpu_cuda_tsb.out \
	    _ref/pfsp_multigpu_cuda_tsb.out _ref/cbase_layout.txt

.PHONY: all clean

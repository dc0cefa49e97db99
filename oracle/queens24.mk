# oracle/queens24.mk — the N-Queens checkers of a MAX_QUEENS = 24 build (boards of 21..24 queens, 25-byte nodes);
# TEST INFRASTRUCTURE, like everything under oracle/ (oracle/pyoracle24.py runs it).
#
#   make -f queens24.mk          -> liboracle24.so           our C restatement (tsb_oracle.c) as `chpl -sMAX_QUEENS=24`
#   make -f queens24.mk ref      -> _ref/libref_nqueens24.so  the reference's own C sources with MAX_QUEENS 24
#
# Neither tsb_oracle.h (OR_MAX_QUEENS, :27) nor the reference's baselines/nqueens/lib/NQueens_node.h (MAX_QUEENS, :10)
# guards its constant with #ifndef, and both are included by quoted name from their sources' own directory: each build
# works on a scratch copy under _ref/ (a build artefact, git-ignored) with that one line rewritten by sed and checked by
# grep, as oracle/Makefile does for MAX_JOBS = 50.
TSB200_REFERENCE ?= $(abspath $(CURDIR)/../../reference)
REF ?= $(TSB200_REFERENCE)
CC  ?= gcc
CFLAGS_OR  := -O2 -Wall -Wextra -std=c11 -fPIC
CFLAGS_REF := -O3 -fPIC -w

NQ  := $(REF)/baselines/nqueens
COM := $(REF)/baselines/commons
O24 := _ref/oracle24
Q24 := _ref/queens24/nqueens

all: liboracle24.so

liboracle24.so: tsb_oracle.c tsb_oracle.h taillard_data.inc
	mkdir -p $(O24)
	cp tsb_oracle.c tsb_oracle.h taillard_data.inc $(O24)/
	sed -i 's/^#define OR_MAX_QUEENS 20 /#define OR_MAX_QUEENS 24 /' $(O24)/tsb_oracle.h
	grep -q '^#define OR_MAX_QUEENS 24 ' $(O24)/tsb_oracle.h
	$(CC) $(CFLAGS_OR) -shared -o $@ $(O24)/tsb_oracle.c

ref: _ref/libref_nqueens24.so

_ref/queens24/.stamp:
	mkdir -p $(Q24)/lib _ref/queens24/commons
	cp $(NQ)/nqueens_c.c $(Q24)/
	cp $(NQ)/lib/NQueens_node.* $(NQ)/lib/Pool.* $(Q24)/lib/
	cp $(COM)/util.* _ref/queens24/commons/
	sed -i 's/^#define MAX_QUEENS 20/#define MAX_QUEENS 24/' $(Q24)/lib/NQueens_node.h
	grep -q '^#define MAX_QUEENS 24' $(Q24)/lib/NQueens_node.h
	touch $@
# `main` renamed and oracle/ref_batch.c around the reference's isSafe / decompose / Pool, as for libref_nqueens.so
_ref/libref_nqueens24.so: ref_batch.c _ref/queens24/.stamp
	$(CC) $(CFLAGS_REF) -shared -Dmain=ref_nqueens_main -DREF_BATCH_NQUEENS -I$(Q24) -o $@ $(Q24)/nqueens_c.c \
	    $(Q24)/lib/NQueens_node.c $(Q24)/lib/Pool.c _ref/queens24/commons/util.c ref_batch.c

clean:
	rm -rf liboracle24.so $(O24) _ref/queens24 _ref/libref_nqueens24.so

.PHONY: all ref clean

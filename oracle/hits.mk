# oracle/hits.mk -- builds the HITS CHECKER (test infrastructure, never product code);
# `make -C oracle -f hits.mk all`, run by __graft_entry__.build() after oracle/wsp.mk.
#
#   oracle -> oracle/_build/libhits_oracle.so   plain-C restatement of cuGraph's HITS (cugraph_hits_oracle.c).  cuGraph
#                                               is third party and absent from the reference checkout, so the
#                                               restatement is pinned by the fixtures in tests/golden/hits_e2e.json.
HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC        ?= gcc

.PHONY: all oracle
all: oracle

oracle: $(HERE)_build/libhits_oracle.so

$(HERE)_build/libhits_oracle.so: $(HERE)cugraph_hits_oracle.c
	mkdir -p $(HERE)_build
	$(CC) -std=c11 -O2 -ffp-contract=off -fPIC -shared -o $@ $(HERE)cugraph_hits_oracle.c -lm

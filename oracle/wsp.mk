# oracle/wsp.mk -- builds the weighted-shortest-path CHECKER (test infrastructure, never product code);
# `make -C oracle -f wsp.mk all`, run by __graft_entry__.build() after oracle/biconnectivity.mk.
#
#   oracle -> oracle/_build/libwsp_oracle.so   plain-C restatement of the engine's cursor (wsp_oracle.c).  The engine
#                                              operator cannot be compiled on its own, so the reference's behaviour is
#                                              pinned by the fixtures in tests/golden/wsp_unit_cases.json instead.
HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC        ?= gcc

.PHONY: all oracle
all: oracle

oracle: $(HERE)_build/libwsp_oracle.so

# -fno-fast-math / -ffp-contract=off: every total is one IEEE round-to-nearest addition, as in the engine
$(HERE)_build/libwsp_oracle.so: $(HERE)wsp_oracle.c
	mkdir -p $(HERE)_build
	$(CC) -std=c11 -O2 -ffp-contract=off -fPIC -shared -o $@ $(HERE)wsp_oracle.c -lm

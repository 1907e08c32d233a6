# oracle/scc.mk -- builds the strongly-connected-components CHECKER (test infrastructure, never product code);
# `make -C oracle -f scc.mk all`, run by __graft_entry__.build() after oracle/bipartite.mk.
#
#   oracle -> oracle/_build/libscc_oracle.so   iterative Tarjan (scc_oracle.c), always buildable
# There is no reference module to compile: the reference computes these components in Python, through networkx
# (query_modules/nxalg.py); tests/golden/scc_cases.json records networkx's answers instead.
HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC        ?= gcc

.PHONY: all oracle
all: oracle

oracle: $(HERE)_build/libscc_oracle.so

$(HERE)_build/libscc_oracle.so: $(HERE)scc_oracle.c
	mkdir -p $(HERE)_build
	$(CC) -std=c11 -O2 -fPIC -shared -o $@ $(HERE)scc_oracle.c

# oracle/bipartite.mk -- builds the maximum bipartite matching CHECKERS (test infrastructure, never product code);
# `make -C oracle -f bipartite.mk all`, run by __graft_entry__.build() after oracle/hits.mk.
#
#   oracle -> oracle/_build/libbipartite_oracle.so                 plain-C colouring + iterative Hopcroft-Karp
#                                                                  (bipartite_oracle.c), always buildable
#   ref    -> oracle/_ref/bipartite_matching_reference.so          the reference's unmodified query module, compiled IN
#                                                                  PLACE from $(REFERENCE); skipped when it is absent.
REFERENCE ?= /root/reference
BM_DIR    := $(REFERENCE)/mage/cpp/bipartite_matching_module
HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC        ?= gcc
CXX       ?= g++

.PHONY: all oracle ref
all: oracle ref

oracle: $(HERE)_build/libbipartite_oracle.so

$(HERE)_build/libbipartite_oracle.so: $(HERE)bipartite_oracle.c
	mkdir -p $(HERE)_build
	$(CC) -std=c11 -O2 -fPIC -shared -o $@ $(HERE)bipartite_oracle.c

ifneq ($(wildcard $(BM_DIR)/bipartite_matching_module.cpp),)
ref: $(HERE)_ref/bipartite_matching_reference.so

# its undefined mgp_* symbols bind to the host that loads it (tests/mgp_wcc_host.cpp)
$(HERE)_ref/bipartite_matching_reference.so: $(BM_DIR)/bipartite_matching_module.cpp \
                                             $(BM_DIR)/algorithm/bipartite_matching.cpp
	mkdir -p $(HERE)_ref
	$(CXX) -std=c++20 -O2 -fPIC -shared -w -I$(REFERENCE)/include -I$(BM_DIR) -o $@ $^
else
ref:
	@echo "oracle/bipartite.mk: $(REFERENCE) not present -- keeping prebuilt oracle/_ref/ (if any)"
endif

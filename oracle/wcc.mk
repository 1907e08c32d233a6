# oracle/wcc.mk -- builds the weakly-connected-components CHECKERS (test infrastructure, never product code);
# `make -C oracle -f wcc.mk all`, run by __graft_entry__.build() after oracle/betweenness.mk.
#
#   oracle -> oracle/_build/libwcc_oracle.so                        plain-C restatement (wcc_oracle.c), always buildable
#   ref    -> oracle/_ref/weakly_connected_components_reference.so  the reference's unmodified query module, compiled IN
#                                                                   PLACE from $(REFERENCE); skipped when it is absent.
REFERENCE ?= /root/reference
WCC_DIR   := $(REFERENCE)/mage/cpp/connectivity_module
HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC        ?= gcc
CXX       ?= g++

.PHONY: all oracle ref
all: oracle ref

oracle: $(HERE)_build/libwcc_oracle.so

$(HERE)_build/libwcc_oracle.so: $(HERE)wcc_oracle.c
	mkdir -p $(HERE)_build
	$(CC) -std=c11 -O2 -fPIC -shared -o $@ $(HERE)wcc_oracle.c

ifneq ($(wildcard $(WCC_DIR)/connectivity_module.cpp),)
ref: $(HERE)_ref/weakly_connected_components_reference.so

# its undefined mgp_* symbols bind to the host that loads it (tests/mgp_wcc_host.cpp)
$(HERE)_ref/weakly_connected_components_reference.so: $(WCC_DIR)/connectivity_module.cpp
	mkdir -p $(HERE)_ref
	$(CXX) -std=c++20 -O2 -fPIC -shared -w -I$(REFERENCE)/include -o $@ $(WCC_DIR)/connectivity_module.cpp
else
ref:
	@echo "oracle/wcc.mk: $(REFERENCE) not present -- keeping prebuilt oracle/_ref/ (if any)"
endif

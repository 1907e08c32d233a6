# oracle/biconnectivity.mk -- builds the bridges / biconnected components CHECKERS (test infrastructure, never product
# code); `make -C oracle -f biconnectivity.mk all`, run by __graft_entry__.build() after oracle/wcc.mk.
#
#   oracle -> oracle/_build/libbiconnectivity_oracle.so           plain-C iterative Hopcroft-Tarjan
#                                                                 (biconnectivity_oracle.c), always buildable
#   ref    -> oracle/_ref/bridges_reference.so                    the reference's unmodified query modules, compiled IN
#             oracle/_ref/biconnected_components_reference.so     PLACE from $(REFERENCE); skipped when it is absent.
REFERENCE ?= /root/reference
BRIDGES_DIR := $(REFERENCE)/mage/cpp/bridges_module
BCC_DIR     := $(REFERENCE)/mage/cpp/biconnected_components_module
HERE        := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CC          ?= gcc
CXX         ?= g++

.PHONY: all oracle ref
all: oracle ref

oracle: $(HERE)_build/libbiconnectivity_oracle.so

$(HERE)_build/libbiconnectivity_oracle.so: $(HERE)biconnectivity_oracle.c
	mkdir -p $(HERE)_build
	$(CC) -std=c11 -O2 -fPIC -shared -o $@ $(HERE)biconnectivity_oracle.c

ifneq ($(wildcard $(BRIDGES_DIR)/bridges_module.cpp),)
ref: $(HERE)_ref/bridges_reference.so $(HERE)_ref/biconnected_components_reference.so

# their undefined mgp_* symbols bind to the host that loads them (tests/mgp_edge_host.cpp)
$(HERE)_ref/bridges_reference.so: $(BRIDGES_DIR)/bridges_module.cpp $(BRIDGES_DIR)/algorithm/bridges.cpp
	mkdir -p $(HERE)_ref
	$(CXX) -std=c++20 -O2 -fPIC -shared -w -I$(REFERENCE)/include -o $@ $^

$(HERE)_ref/biconnected_components_reference.so: $(BCC_DIR)/biconnected_components_module.cpp \
                                                 $(BCC_DIR)/algorithm/biconnected_components.cpp
	mkdir -p $(HERE)_ref
	$(CXX) -std=c++20 -O2 -fPIC -shared -w -I$(REFERENCE)/include -o $@ $^
else
ref:
	@echo "oracle/biconnectivity.mk: $(REFERENCE) not present -- keeping prebuilt oracle/_ref/ (if any)"
endif

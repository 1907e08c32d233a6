// memgraph_b200/csrc/bipartite_matching_module.cpp -- the drop-in `bipartite_matching` query module (host side).
//
// Replaces the procedure `max` of mage/cpp/bipartite_matching_module/bipartite_matching_module.cpp behind the same ABI:
//   CALL bipartite_matching.max() YIELD maximum_bipartite_matching                          (reference :45-55)
// Same procedure and field names and types.  The graph view is mg_utility::GetGraphView's (include/mg_utils.hpp):
// every vertex becomes a node, an out-edge is kept only if both endpoints are nodes of the view.  The result is always
// exactly one row: 0 for an empty view or a view without edges (without touching the device), 0 when the view has a
// self-loop or an odd cycle, otherwise the size of a maximum matching (bipartite_matching.cu).
// Difference not reproduced: the reference narrows the count to `int`; here it keeps 64 bits.  A graph with 32-bit
// dense ids has at most 2^31 - 1 pairs, so the value is the same.
#include <cstdint>

#include "mgb200_bfs.h"
#include "mgb200_pagerank.h"
#include "mgp_module_common.hpp"

using namespace mgb200_module;

namespace {

constexpr const char *kProcedureMax = "max";
constexpr const char *kFieldMatchingNumber = "maximum_bipartite_matching";

void Max(mgp_list * /*args*/, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  const HostGraph hg = PullGraph(graph, memory, UnknownGid::kUnknownDropped);
  int64_t matched = 0;
  if (!hg.from.empty()) {
    const BfsDeviceGraph dg(hg);
    mgb200_matching_stats stats{};
    CheckDevice(mgb200_bipartite_matching_run(dg.graph.h, MustAbortPoll, graph, nullptr, nullptr, &stats));
    matched = static_cast<int64_t>(stats.matched);
  }
  InsertColumns(NewRecord(result), memory, kFieldMatchingNumber, matched);
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) int mgp_init_module(struct mgp_module *module, struct mgp_memory * /*memory*/) {
  try {
    mgp_proc *proc = nullptr;
    Check(mgp_module_add_read_procedure(module, kProcedureMax, Guarded<Max>, &proc));
    mgp_type *type_int = nullptr;
    Check(mgp_type_int(&type_int));
    Check(mgp_proc_add_result(proc, kFieldMatchingNumber, type_int));
  } catch (...) {
    return 1;
  }
  return 0;
}

__attribute__((visibility("default"))) int mgp_shutdown_module(void) { return 0; }

}  // extern "C"

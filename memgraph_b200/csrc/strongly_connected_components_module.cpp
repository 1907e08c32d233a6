// memgraph_b200/csrc/strongly_connected_components_module.cpp -- the `strongly_connected_components` query module
// (host side).
//
//   CALL strongly_connected_components.get() YIELD node, component_id
// The partition is the reference's nxalg.strongly_connected_components (query_modules/nxalg.py), networkx's strongly
// connected components of the MultiDiGraph of the graph view (scc.cu).  The graph view is mg_utility::GetGraphView's
// (include/mg_utils.hpp): every vertex becomes a node, dense id = visit order, an out-edge is kept only if both
// endpoints are nodes of the view.  Components are numbered in the order their first vertex appears in that visit
// order; every node gets a row, isolated ones included, and self-loops and multi-edges change nothing.  Rows: one per
// node in dense order; a vertex that has vanished is skipped in analytical mode (its component number stays used) and
// is "Invalid ID!" in transactional mode, as in weakly_connected_components.  An empty view yields zero rows without
// touching the device.  The host's abort flag is polled between the device's round trips.
// The one difference from nxalg: nxalg returns a single row holding a list of vertex lists; here every node has its
// own (node, component_id) row.  This Cypher rebuilds nxalg's shape:
//   CALL strongly_connected_components.get() YIELD node, component_id
//   WITH component_id, collect(node) AS c RETURN collect(c) AS components
#include <cstdint>
#include <vector>

#include "mgb200_bfs.h"
#include "mgb200_pagerank.h"
#include "mgp_module_common.hpp"

using namespace mgb200_module;

namespace {

constexpr const char *kProcedureGet = "get";
constexpr const char *kFieldComponentId = "component_id";

void Strong(mgp_list * /*args*/, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  const HostGraph hg = PullGraph(graph, memory, UnknownGid::kUnknownDropped);
  const uint64_t n = hg.gid_of_dense.size();
  std::vector<int64_t> component(n, 0);
  if (n != 0) {
    const BfsDeviceGraph dg(hg);
    CheckDevice(mgb200_scc_run(dg.graph.h, MustAbortPoll, graph, component.data(), nullptr));
  }

  if (mgp_result_reserve != nullptr && n != 0) (void)mgp_result_reserve(result, n);
  for (uint64_t dense = 0; dense < n; ++dense)
    EmitNodeRow(graph, result, memory, hg.gid_of_dense[dense], kFieldComponentId, component[dense]);
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) int mgp_init_module(struct mgp_module *module, struct mgp_memory * /*memory*/) {
  try {
    mgp_proc *proc = nullptr;
    Check(mgp_module_add_read_procedure(module, kProcedureGet, Guarded<Strong>, &proc));
    mgp_type *type_node = nullptr, *type_int = nullptr;
    Check(mgp_type_node(&type_node));
    Check(mgp_type_int(&type_int));
    Check(mgp_proc_add_result(proc, kFieldNode, type_node));
    Check(mgp_proc_add_result(proc, kFieldComponentId, type_int));
  } catch (...) {
    return 1;
  }
  return 0;
}

__attribute__((visibility("default"))) int mgp_shutdown_module(void) { return 0; }

}  // extern "C"

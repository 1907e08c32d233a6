// memgraph_b200/csrc/weakly_connected_components_module.cpp -- the drop-in `weakly_connected_components` query module
// (host side).
//
// Replaces the procedure `get` of mage/cpp/connectivity_module/connectivity_module.cpp behind the same ABI:
//   CALL weakly_connected_components.get() YIELD node, component_id                          (reference :88-99)
// Same procedure and field names, types and registration order.  The graph view is mg_utility::GetGraphView's
// (include/mg_utils.hpp:127-171): every vertex becomes a node, dense id = visit order, an out-edge is kept only if both
// endpoints are nodes of the view (mg_graph.hpp:213-217).  Components are numbered in the order their first vertex
// appears in that visit order (the reference's BFS loop, :45-72); every node gets a row, isolated ones included, and
// self-loops and multi-edges change nothing.  Rows: one per node in dense order; a vertex that has vanished is skipped
// in analytical mode (its component number stays used) and is "Invalid ID!" in transactional mode, like
// mg_utility::GetNodeForInsertion.  An empty view yields zero rows without touching the device.
// Differences not reproduced:
//   * the reference emits its rows in unordered_map order, which is unspecified; here they come in dense order;
//   * the reference narrows node ids and component ids to `int` (:76-77); here both keep 64 bits.
#include <cstdint>
#include <cstdlib>
#include <exception>
#include <string>
#include <vector>

#include "mgb200_bfs.h"
#include "mgb200_pagerank.h"
#include "mgp_module_common.hpp"

using namespace mgb200_module;

namespace {

constexpr const char *kProcedureGet = "get";
constexpr const char *kFieldComponentId = "component_id";

void Weak(mgp_list * /*args*/, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  const HostGraph hg = PullGraph(graph, memory, UnknownGid::kUnknownDropped);
  const uint64_t n = hg.gid_of_dense.size();
  std::vector<int64_t> component(n, 0);
  if (n != 0) {
    const BfsDeviceGraph dg(hg);
    CheckDevice(mgb200_wcc_run(dg.graph.h, component.data(), nullptr));
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
    Check(mgp_module_add_read_procedure(module, kProcedureGet, Guarded<Weak>, &proc));
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

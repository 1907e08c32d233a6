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
constexpr const char *kFieldVertex = "node";
constexpr const char *kFieldComponentId = "component_id";

void EmitRecord(mgp_graph *graph, mgp_result *result, mgp_memory *memory, int64_t gid, int64_t component_id) {
  mgp_vertex *vertex = nullptr;
  Check(mgp_graph_get_vertex_by_id(graph, mgp_vertex_id{gid}, memory, &vertex));
  if (vertex == nullptr) {
    int transactional = 0;
    Check(mgp_graph_is_transactional(graph, &transactional));
    if (transactional) throw ModuleError("Invalid ID!");
    return;
  }
  OwnedValue node;
  Check(mgp_value_make_vertex(vertex, &node.v));  // takes ownership of `vertex` on success
  mgp_result_record *record = nullptr;
  Check(mgp_result_new_record(result, &record));
  if (record == nullptr)
    throw ModuleError("Not enough memory! For more details please visit https://memgr.ph/memory-control");
  Check(mgp_result_record_insert(record, kFieldVertex, node.v));
  OwnedValue value;
  Check(mgp_value_make_int(component_id, memory, &value.v));
  Check(mgp_result_record_insert(record, kFieldComponentId, value.v));
}

void Weak(mgp_list * /*args*/, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  try {
    const HostGraph hg = PullGraph(graph, memory, UnknownGid::kUnknownDropped);
    const uint64_t n = hg.gid_of_dense.size();
    std::vector<int64_t> component(n, 0);
    if (n != 0) {
      const char *dev_env = std::getenv("MGB200_DEVICE");
      const std::vector<uint64_t> from64(hg.from.begin(), hg.from.end()), to64(hg.to.begin(), hg.to.end());
      mgb200_bfs_graph *dg = nullptr;
      if (mgb200_bfs_graph_create_host(dev_env ? std::atoi(dev_env) : 0, n, from64.size(), from64.data(), to64.data(),
                                       &dg) != MGB200_OK)
        throw ModuleError(mgb200_last_error());
      const int rc = mgb200_wcc_run(dg, component.data(), nullptr);
      const std::string message = rc != MGB200_OK ? mgb200_last_error() : "";
      mgb200_bfs_graph_destroy(dg);
      if (rc != MGB200_OK) throw ModuleError(message);
    }

    if (mgp_result_reserve != nullptr && n != 0) (void)mgp_result_reserve(result, n);
    for (uint64_t dense = 0; dense < n; ++dense) EmitRecord(graph, result, memory, hg.gid_of_dense[dense], component[dense]);
  } catch (const std::exception &e) {
    (void)mgp_result_set_error_msg(result, e.what());  // nothing may escape the callback (reference :79-83)
  } catch (...) {
    (void)mgp_result_set_error_msg(result, "Unknown exception!");
  }
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) int mgp_init_module(struct mgp_module *module, struct mgp_memory * /*memory*/) {
  try {
    mgp_proc *proc = nullptr;
    Check(mgp_module_add_read_procedure(module, kProcedureGet, Weak, &proc));
    mgp_type *type_node = nullptr, *type_int = nullptr;
    Check(mgp_type_node(&type_node));
    Check(mgp_type_int(&type_int));
    Check(mgp_proc_add_result(proc, kFieldVertex, type_node));
    Check(mgp_proc_add_result(proc, kFieldComponentId, type_int));
  } catch (...) {
    return 1;
  }
  return 0;
}

__attribute__((visibility("default"))) int mgp_shutdown_module(void) { return 0; }

}  // extern "C"

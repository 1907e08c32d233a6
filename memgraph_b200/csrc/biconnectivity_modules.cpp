// memgraph_b200/csrc/biconnectivity_modules.cpp -- the drop-in `bridges` and `biconnected_components` query modules
// (host side).  Compiled twice (memgraph_b200/build.py):
//   -DMGB200_BRIDGES=1 -> bridges.so                 CALL bridges.get() YIELD node_from, node_to
//        (mage/cpp/bridges_module/bridges_module.cpp:39-69)
//   -DMGB200_BRIDGES=0 -> biconnected_components.so  CALL biconnected_components.get() YIELD bcc_id, node_from, node_to
//        (mage/cpp/biconnected_components_module/biconnected_components_module.cpp:43-83)
// Same procedure and field names, types and registration order.  The graph view is mg_utility::GetGraphView's
// (include/mg_utils.hpp:127-171) as an undirected multigraph: every vertex becomes a node, dense id = visit order, an
// out-edge is kept only if both endpoints are nodes of the view (mg_graph.hpp:213-217), and each edge is in both
// endpoints' lists.  The device computes the multigraph's bridges and biconnected components (mgb200_biconnectivity_run).
//   bridges                 one row per bridge, in its stored direction (from, to), in view edge order.  An edge with
//                           a parallel copy is never a bridge, nor is a self-loop (bridges.cpp:47-50)
//   biconnected_components  one row per non-loop edge, rows grouped by ascending bcc_id, view edge order inside a
//                           component; components are numbered in the order of their first edge in view edge order
// A vertex that has vanished skips the row in analytical mode and is "Invalid ID!" in transactional mode, like
// mg_utility::GetNodeForInsertion.  An empty view yields zero rows without touching the device.
// Differences not reproduced:
//   * the reference emits rows in DFS order and numbers components in DFS pop order, which depend on adjacency order;
//     its own tests compare components as sets of edges (biconnected_components_test.cpp:26-51);
//   * the reference narrows node ids to `int` (bridges_module.cpp:27-28, biconnected_components_module.cpp:56); here
//     ids keep 64 bits;
//   * the reference drops every copy of an edge that runs parallel to a DFS tree edge but the one the DFS walked down
//     (biconnected_components.cpp:43-45); here every non-loop edge gets its row.
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <exception>
#include <string>
#include <vector>

#include "mgb200_bfs.h"
#include "mgb200_pagerank.h"
#include "mgp_module_common.hpp"

#ifndef MGB200_BRIDGES
#define MGB200_BRIDGES 1
#endif

using namespace mgb200_module;

namespace {

constexpr const char *kProcedureGet = "get";
constexpr const char *kFieldBccId = "bcc_id";
constexpr const char *kFieldNodeFrom = "node_from";
constexpr const char *kFieldNodeTo = "node_to";

void EmitRecord(mgp_graph *graph, mgp_result *result, mgp_memory *memory, int64_t from_gid, int64_t to_gid,
                const int64_t *bcc_id) {
  OwnedValue from, to;
  if (!NodeValue(graph, memory, from_gid, &from) || !NodeValue(graph, memory, to_gid, &to)) return;
  mgp_result_record *record = NewRecord(result);
  if (bcc_id) {
    OwnedValue value;
    Check(mgp_value_make_int(*bcc_id, memory, &value.v));
    Check(mgp_result_record_insert(record, kFieldBccId, value.v));
  }
  Check(mgp_result_record_insert(record, kFieldNodeFrom, from.v));
  Check(mgp_result_record_insert(record, kFieldNodeTo, to.v));
}

void Get(mgp_list * /*args*/, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  const HostGraph hg = PullGraph(graph, memory, UnknownGid::kUnknownDropped);
  const uint64_t n = hg.gid_of_dense.size(), m = hg.from.size();
  if (n == 0) return;
  std::vector<uint8_t> bridge(m, 0);
  std::vector<int64_t> bcc(m, -1);
  {
    const BfsDeviceGraph dg(hg);
    CheckDevice(mgb200_biconnectivity_run(dg.graph.h, m, dg.from.data(), dg.to.data(),
                                          MGB200_BRIDGES ? bridge.data() : nullptr, MGB200_BRIDGES ? nullptr : bcc.data(),
                                          nullptr));
  }
#if MGB200_BRIDGES
  for (uint64_t e = 0; e < m; ++e)
    if (bridge[e]) EmitRecord(graph, result, memory, hg.gid_of_dense[hg.from[e]], hg.gid_of_dense[hg.to[e]], nullptr);
#else
  // a stable counting sort of the non-loop edges by component: ascending bcc_id, view edge order inside
  int64_t components = 0;
  for (uint64_t e = 0; e < m; ++e) components = std::max(components, bcc[e] + 1);
  std::vector<uint64_t> start(components + 1, 0);
  for (uint64_t e = 0; e < m; ++e)
    if (bcc[e] >= 0) ++start[bcc[e] + 1];
  for (int64_t c = 0; c < components; ++c) start[c + 1] += start[c];
  std::vector<uint64_t> rows(start[components]);
  for (uint64_t e = 0; e < m; ++e)
    if (bcc[e] >= 0) rows[start[bcc[e]]++] = e;
  if (mgp_result_reserve != nullptr && !rows.empty()) (void)mgp_result_reserve(result, rows.size());
  for (const uint64_t e : rows)
    EmitRecord(graph, result, memory, hg.gid_of_dense[hg.from[e]], hg.gid_of_dense[hg.to[e]], &bcc[e]);
#endif
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) int mgp_init_module(struct mgp_module *module, struct mgp_memory * /*memory*/) {
  try {
    mgp_proc *proc = nullptr;
    Check(mgp_module_add_read_procedure(module, kProcedureGet, Guarded<Get>, &proc));
    mgp_type *type_node = nullptr;
    Check(mgp_type_node(&type_node));
    if (!MGB200_BRIDGES) {
      mgp_type *type_int = nullptr;
      Check(mgp_type_int(&type_int));
      Check(mgp_proc_add_result(proc, kFieldBccId, type_int));
    }
    Check(mgp_proc_add_result(proc, kFieldNodeFrom, type_node));
    Check(mgp_proc_add_result(proc, kFieldNodeTo, type_node));
  } catch (...) {
    return 1;
  }
  return 0;
}

__attribute__((visibility("default"))) int mgp_shutdown_module(void) { return 0; }

}  // extern "C"

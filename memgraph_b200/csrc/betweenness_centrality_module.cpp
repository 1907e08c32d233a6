// memgraph_b200/csrc/betweenness_centrality_module.cpp -- the drop-in `betweenness_centrality` query module (host side).
//
// Replaces the procedure `get` of mage/cpp/betweenness_centrality_module/betweenness_centrality_module.cpp behind the
// same ABI:
//   CALL betweenness_centrality.get(directed = true, normalized = true, threads = <hardware threads>)
//   YIELD node, betweenness_centrality                                                      (reference :71-105)
// Same procedure / argument / field names, types, defaults and registration order.  `threads` only sizes the
// reference's CPU thread pool and never changes its result; it is read and ignored here (values <= 0 are no error in
// the reference either, :47-49).  The graph view is mg_utility::GetGraphView's (include/mg_utils.hpp:127-171): every
// vertex becomes a node, dense id = visit order, an out-edge is kept only if both endpoints are nodes of the view
// (mg_graph.hpp:213-217); `directed = false` walks every edge from both ends.  Rows: one per node in dense order; a
// vertex that has vanished is skipped in analytical mode and is "Invalid ID!" in transactional mode, like
// mg_utility::GetNodeForInsertion.  (The reference narrows the id to `int` on that call (:59) -- not reproduced.)
#include <cstdint>
#include <cstdlib>
#include <exception>
#include <string>
#include <thread>
#include <vector>

#include "mgb200_bfs.h"
#include "mgb200_pagerank.h"
#include "mgp_module_common.hpp"

using namespace mgb200_module;

namespace {

constexpr const char *kProcedureGet = "get";
constexpr const char *kArgumentDirected = "directed";
constexpr const char *kArgumentNormalized = "normalized";
constexpr const char *kArgumentThreads = "threads";
constexpr const char *kFieldBCScore = "betweenness_centrality";

void GetBetweennessCentrality(mgp_list *args, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  mgp_value *arg = nullptr;
  int directed = 0, normalized = 0;
  int64_t threads = 0;
  Check(mgp_list_at(args, 0, &arg));
  Check(mgp_value_get_bool(arg, &directed));
  Check(mgp_list_at(args, 1, &arg));
  Check(mgp_value_get_bool(arg, &normalized));
  Check(mgp_list_at(args, 2, &arg));
  Check(mgp_value_get_int(arg, &threads));
  (void)threads;

  const HostGraph hg = PullGraph(graph, memory, UnknownGid::kUnknownDropped);
  const uint64_t n = hg.gid_of_dense.size();
  std::vector<double> bc(n, 0.0);
  if (n != 0) {  // an empty view yields zero rows in the reference too; nothing to compute anywhere
    const BfsDeviceGraph dg(hg);
    CheckDevice(mgb200_bc_run(dg.graph.h, directed != 0, 0, n, MustAbortPoll, graph, bc.data(), 0, nullptr));
    if (normalized) {  // betweenness_centrality.cpp:138-143; (n - 1) * (n - 2) in uint64_t
      const uint64_t pairs = (n - 1) * (n - 2);
      const double constant = n > 2 ? (directed ? 1.0 : 2.0) / static_cast<double>(pairs) : 1.0;
      for (double &value : bc) value *= constant;
    }
  }

  if (mgp_result_reserve != nullptr && n != 0) (void)mgp_result_reserve(result, n);
  for (uint64_t dense = 0; dense < n; ++dense)
    EmitNodeRow(graph, result, memory, hg.gid_of_dense[dense], kFieldBCScore, bc[dense]);
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) int mgp_init_module(struct mgp_module *module, struct mgp_memory *memory) {
  OwnedValue default_directed, default_normalized, default_threads;  // destroyed on every path (reference :92-102)
  try {
    mgp_proc *proc = nullptr;
    Check(mgp_module_add_read_procedure(module, kProcedureGet, Guarded<GetBetweennessCentrality>, &proc));
    Check(mgp_value_make_bool(1, memory, &default_directed.v));
    Check(mgp_value_make_bool(1, memory, &default_normalized.v));
    Check(mgp_value_make_int(static_cast<int64_t>(std::thread::hardware_concurrency()), memory, &default_threads.v));
    mgp_type *type_bool = nullptr, *type_int = nullptr, *type_node = nullptr, *type_float = nullptr;
    Check(mgp_type_bool(&type_bool));
    Check(mgp_type_int(&type_int));
    Check(mgp_type_node(&type_node));
    Check(mgp_type_float(&type_float));
    Check(mgp_proc_add_opt_arg(proc, kArgumentDirected, type_bool, default_directed.v));
    Check(mgp_proc_add_opt_arg(proc, kArgumentNormalized, type_bool, default_normalized.v));
    Check(mgp_proc_add_opt_arg(proc, kArgumentThreads, type_int, default_threads.v));
    Check(mgp_proc_add_result(proc, kFieldNode, type_node));
    Check(mgp_proc_add_result(proc, kFieldBCScore, type_float));
  } catch (...) {
    return 1;
  }
  return 0;
}

__attribute__((visibility("default"))) int mgp_shutdown_module(void) { return 0; }

}  // extern "C"

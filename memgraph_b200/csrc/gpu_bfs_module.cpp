// memgraph_b200/csrc/gpu_bfs_module.cpp -- query module `gpu_bfs`: the engine's breadth-first expansion as a procedure.
//
// In the reference, `MATCH (a)-[*BFS l..u]->(b)` is an engine operator (SingleSourceShortestPathCursor,
// src/query/plan/operator.cpp:2692-2912) with no plugin boundary, so there is nothing to drop in for; this module
// exposes the same arithmetic behind the query-module ABI instead (SURVEY 8f-2):
//
//   CALL gpu_bfs.distances(source, direction = 0, lower_bound = 1, upper_bound = -1) YIELD node, distance
//
//   source      NODE     the vertex the expansion starts from (never produced itself, :2833)
//   direction   INTEGER  0 = OUT, 1 = IN, 2 = BOTH                         (EdgeAtom::Direction)
//   lower_bound INTEGER  minimum depth, default 1                          (:2824-2825)
//   upper_bound INTEGER  maximum depth, -1 = unbounded (the default)       (:2826-2828)
//   -> one row per vertex the cursor would produce, with its BFS depth.
// Edge-type filters and filter lambdas of the Cypher syntax are not expressible here (they are evaluated by the engine).
#include <cstdint>
#include <limits>
#include <vector>

#include "mgb200_bfs.h"
#include "mgb200_pagerank.h"
#include "mgp_module_common.hpp"

using namespace mgb200_module;

namespace {

constexpr const char *kFieldDistance = "distance";

void Distances(mgp_list *args, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  mgp_value *arg = nullptr;
  mgp_vertex *source = nullptr;
  int64_t direction = 0, lower = 1, upper = -1;
  Check(mgp_list_at(args, 0, &arg));
  Check(mgp_value_get_vertex(arg, &source));
  Check(mgp_list_at(args, 1, &arg));
  Check(mgp_value_get_int(arg, &direction));
  Check(mgp_list_at(args, 2, &arg));
  Check(mgp_value_get_int(arg, &lower));
  Check(mgp_list_at(args, 3, &arg));
  Check(mgp_value_get_int(arg, &upper));
  if (direction < MGB200_BFS_OUT || direction > MGB200_BFS_BOTH)
    throw ModuleError("direction must be 0 (OUT), 1 (IN) or 2 (BOTH)");
  if (upper < 0) upper = std::numeric_limits<int64_t>::max();
  mgp_vertex_id source_id{};
  Check(mgp_vertex_get_id(source, &source_id));

  // an edge to a vertex the iterator never showed is dropped here: the reference cursor has no "map it to the first
  // vertex" behaviour (that is a PageRank-module quirk), and a fabricated edge would change distances
  const HostGraph hg = PullGraph(graph, memory, UnknownGid::kUnknownDropped);
  const uint64_t n = hg.gid_of_dense.size();
  uint64_t source_dense = n;
  if (!hg.dense_of_gid.Find(source_id.as_int, &source_dense)) throw ModuleError("Invalid ID!");

  std::vector<int32_t> dist(n);
  {
    const BfsDeviceGraph dg(hg);
    mgb200_bfs_stats stats{};
    CheckDevice(mgb200_bfs_run(dg.graph.h, source_dense, static_cast<int>(direction), lower, upper, dist.data(), 0,
                               &stats));
  }

  for (uint64_t v = 0; v < n; ++v)
    if (dist[v] >= 0) EmitNodeRow(graph, result, memory, hg.gid_of_dense[v], kFieldDistance, dist[v]);
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) int mgp_init_module(struct mgp_module *module, struct mgp_memory *memory) {
  OwnedValue direction, lower, upper;
  try {
    mgp_proc *proc = nullptr;
    Check(mgp_module_add_read_procedure(module, "distances", Guarded<Distances>, &proc));
    mgp_type *type_int = nullptr, *type_node = nullptr;
    Check(mgp_type_int(&type_int));
    Check(mgp_type_node(&type_node));
    Check(mgp_proc_add_arg(proc, "source", type_node));
    Check(mgp_value_make_int(0, memory, &direction.v));
    Check(mgp_value_make_int(1, memory, &lower.v));
    Check(mgp_value_make_int(-1, memory, &upper.v));
    Check(mgp_proc_add_opt_arg(proc, "direction", type_int, direction.v));
    Check(mgp_proc_add_opt_arg(proc, "lower_bound", type_int, lower.v));
    Check(mgp_proc_add_opt_arg(proc, "upper_bound", type_int, upper.v));
    Check(mgp_proc_add_result(proc, kFieldNode, type_node));
    Check(mgp_proc_add_result(proc, kFieldDistance, type_int));
  } catch (...) {
    return 1;
  }
  return 0;
}

__attribute__((visibility("default"))) int mgp_shutdown_module(void) { return 0; }

}  // extern "C"

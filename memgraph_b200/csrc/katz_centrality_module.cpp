// memgraph_b200/csrc/katz_centrality_module.cpp -- the drop-in `katz_centrality` query module, static part (host side).
//
// Replaces the procedure `get` of mage/cpp/katz_centrality_module/katz_centrality_module.cpp behind the same ABI:
//   CALL katz_centrality.get(alpha = 0.2, epsilon = 1e-2) YIELD node, rank          (reference :59-76)
// Same procedure / argument / field names, types and defaults.  The graph is pulled once through the mgp_graph
// iterators the way mg_utility::GetGraphView does (include/mg_utils.hpp:127-171): every vertex becomes a node, an
// out-edge becomes an edge only if BOTH endpoints are nodes of the view (mg_graph.hpp:213-217 drops it otherwise).
// The reference keys every per-vertex quantity by Memgraph id and walks the active set -- a std::set of those ids
// -- in ascending id order (katz.cpp:174-177), so dense id = rank of the gid in ascending order here: the tie order of
// the convergence test is then the reference's, whatever order the host iterates vertices in.
// Rows: one per vertex of the view, ascending id (the reference emits in unordered_map order, i.e. unspecified);
// a vertex that has vanished is skipped in analytical mode and is "Invalid ID!" in transactional mode, like
// mg_utility::GetNodeForInsertion.  (The reference narrows the id to `int` on that call (:47) -- not reproduced.)
// The online procedures (katz_centrality_online.*) keep state between calls and are not part of this path.
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <exception>
#include <string>
#include <vector>

#include "mgb200_katz.h"
#include "mgp_module_common.hpp"

using namespace mgb200_module;

namespace {

constexpr const char *kProcedureGet = "get";
constexpr const char *kArgumentAlpha = "alpha";
constexpr const char *kArgumentEpsilon = "epsilon";
constexpr const char *kFieldRank = "rank";

struct ViewGraph {
  std::vector<int64_t> gid_of_dense;  // ascending
  std::vector<uint64_t> from, to;     // dense endpoints of the edges whose endpoints both are nodes
};

ViewGraph PullGraphView(mgp_graph *graph, mgp_memory *memory) {
  ViewGraph vg;
  std::size_t approx_vertices = 0, approx_edges = 0;
  Check(mgp_graph_approximate_vertex_count(graph, &approx_vertices));
  Check(mgp_graph_approximate_edge_count(graph, &approx_edges));
  std::vector<int64_t> from_gid, to_gid;
  vg.gid_of_dense.reserve(approx_vertices);
  from_gid.reserve(approx_edges);
  to_gid.reserve(approx_edges);
  {
    VerticesIt vertices(graph, memory);
    std::size_t visited = 0;
    for (mgp_vertex *source = vertices.Get(); source != nullptr; source = vertices.Next(), ++visited) {
      mgp_vertex_id source_id{};
      Check(mgp_vertex_get_id(source, &source_id));
      vg.gid_of_dense.push_back(source_id.as_int);
      OutEdgesIt edges(source, memory);
      for (mgp_edge *edge = edges.Get(); edge != nullptr; edge = edges.Next()) {
        mgp_vertex *destination = nullptr;
        Check(mgp_edge_get_to(edge, &destination));
        mgp_vertex_id destination_id{};
        Check(mgp_vertex_get_id(destination, &destination_id));
        from_gid.push_back(source_id.as_int);
        to_gid.push_back(destination_id.as_int);
      }
      if ((visited & 0xFFF) == 0 && MustAbort(graph)) throw ModuleError("katz_centrality.get aborted by the host");
    }
  }
  std::sort(vg.gid_of_dense.begin(), vg.gid_of_dense.end());
  vg.gid_of_dense.erase(std::unique(vg.gid_of_dense.begin(), vg.gid_of_dense.end()), vg.gid_of_dense.end());
  auto dense_of = [&vg](int64_t gid, uint64_t *dense) {
    const auto it = std::lower_bound(vg.gid_of_dense.begin(), vg.gid_of_dense.end(), gid);
    if (it == vg.gid_of_dense.end() || *it != gid) return false;
    *dense = static_cast<uint64_t>(it - vg.gid_of_dense.begin());
    return true;
  };
  vg.from.reserve(from_gid.size());
  vg.to.reserve(from_gid.size());
  for (std::size_t e = 0; e < from_gid.size(); ++e) {
    uint64_t f = 0, t = 0;
    if (dense_of(from_gid[e], &f) && dense_of(to_gid[e], &t)) {  // mg_graph.hpp:213-217
      vg.from.push_back(f);
      vg.to.push_back(t);
    }
  }
  return vg;
}

void GetKatzCentrality(mgp_list *args, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  mgp_value *arg = nullptr;
  double alpha = 0.0, epsilon = 0.0;
  Check(mgp_list_at(args, 0, &arg));
  Check(mgp_value_get_double(arg, &alpha));
  Check(mgp_list_at(args, 1, &arg));
  Check(mgp_value_get_double(arg, &epsilon));

  const ViewGraph vg = PullGraphView(graph, memory);
  const uint64_t n = vg.gid_of_dense.size();
  std::vector<double> centralities(n, 0.0);
  uint64_t iterations = 0;
  // max_iterations = 0: like the reference, the loop ends only when the ranking has separated (katz.cpp:250)
  if (n != 0)  // an empty view yields zero rows in the reference too; nothing to compute anywhere
    CheckDevice(mgb200_katz_centrality(n, vg.from.size(), vg.from.data(), vg.to.data(), alpha, epsilon, 0,
                                       centralities.data(), &iterations));

  if (mgp_result_reserve != nullptr && n != 0) (void)mgp_result_reserve(result, n);
  for (uint64_t dense = 0; dense < n; ++dense)
    EmitNodeRow(graph, result, memory, vg.gid_of_dense[dense], kFieldRank, centralities[dense]);
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) int mgp_init_module(struct mgp_module *module, struct mgp_memory *memory) {
  OwnedValue default_alpha, default_epsilon;  // both destroyed on every path (the reference destroys alpha twice, :72-73)
  try {
    mgp_proc *proc = nullptr;
    Check(mgp_module_add_read_procedure(module, kProcedureGet, Guarded<GetKatzCentrality>, &proc));
    Check(mgp_value_make_double(0.2, memory, &default_alpha.v));
    Check(mgp_value_make_double(1e-2, memory, &default_epsilon.v));
    mgp_type *type_float = nullptr, *type_node = nullptr;
    Check(mgp_type_float(&type_float));
    Check(mgp_type_node(&type_node));
    Check(mgp_proc_add_opt_arg(proc, kArgumentAlpha, type_float, default_alpha.v));
    Check(mgp_proc_add_opt_arg(proc, kArgumentEpsilon, type_float, default_epsilon.v));
    Check(mgp_proc_add_result(proc, kFieldNode, type_node));
    Check(mgp_proc_add_result(proc, kFieldRank, type_float));
  } catch (...) {
    return 1;
  }
  return 0;
}

__attribute__((visibility("default"))) int mgp_shutdown_module(void) { return 0; }

}  // extern "C"

// memgraph_b200/csrc/cugraph_modules.cpp -- stand-ins for the reference's cuGraph PageRank and HITS query modules on the
// GPU compute ABI (include/mgb200_personalized.h).  Compiled three times (memgraph_b200/build.py):
//   -DMGB200_CUGRAPH_PERSONALIZED=0 -> cugraph.pagerank.so               CALL cugraph.pagerank.get(max_iterations = 100,
//        damping_factor = 0.85, stop_epsilon = 1e-5, weight_property = "weight") YIELD node, pagerank
//        (mage/cpp/cugraph_module/algorithms/pagerank.cu:60-143)
//   -DMGB200_CUGRAPH_PERSONALIZED=1 -> cugraph.personalized_pagerank.so  CALL cugraph.personalized_pagerank.get(
//        personalization_vertices, personalization_values, max_iterations = 100, damping_factor = 0.85,
//        stop_epsilon = 1e-5, weight_property = "weight") YIELD node, pagerank
//        (mage/cpp/cugraph_module/algorithms/personalized_pagerank.cu:59-215)
//   -DMGB200_CUGRAPH_HITS=1         -> cugraph.hits.so                   CALL cugraph.hits.get(max_iterations = 100,
//        tolerance = 1e-5, normalized = true) YIELD node, hubs, authorities
//        (mage/cpp/cugraph_module/algorithms/hits.cu: unweighted directed view, no initial hub guess)
// Same procedure name, argument names / types / defaults / order and result fields.  Behaviour restated from the
// reference modules: the graph view is weighted (the named edge property when it is a number, else 1.0,
// include/mg_utils.hpp:166); cuGraph only knows vertices that occur in an edge, so isolated vertices get no row, an isolated
// seed is skipped, and with no usable seed the procedure returns no rows (:116-123, :129); list lengths must match
// (:71-73); no seeds -> no rows (:74).  Rows are emitted in ascending vertex id (cuGraph's renumbering order is
// unspecified; the reference's tests sort).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <exception>
#include <stdexcept>
#include <string>
#include <vector>

#include "mgb200_personalized.h"
#include "mgp_module_common.hpp"

#ifndef MGB200_CUGRAPH_PERSONALIZED
#define MGB200_CUGRAPH_PERSONALIZED 0
#endif
#ifndef MGB200_CUGRAPH_HITS
#define MGB200_CUGRAPH_HITS 0
#endif

using namespace mgb200_module;

namespace {

constexpr const char *kProcedureGet = "get";
constexpr const char *kFieldPageRank = "pagerank";
constexpr const char *kFieldHubs = "hubs";
constexpr const char *kFieldAuthorities = "authorities";
constexpr double kDefaultWeight = 1.0;

struct WeightedView {
  std::vector<int64_t> gid_of_dense;  // ascending; only vertices that occur in an edge
  std::vector<uint32_t> from, to;
  std::vector<double> weight;
};

// mg_utility::GetNumericProperty: the property when it is a number, else the default
double EdgeWeight(mgp_edge *edge, const char *property, mgp_memory *memory) {
  mgp_value *value = nullptr;
  Check(mgp_edge_get_property(edge, property, memory, &value));
  OwnedValue owned;
  owned.v = value;
  mgp_value_type type{};
  Check(mgp_value_get_type(value, &type));
  if (type == mgp_value_type::MGP_VALUE_TYPE_DOUBLE) {
    double d = 0.0;
    Check(mgp_value_get_double(value, &d));
    return d;
  }
  if (type == mgp_value_type::MGP_VALUE_TYPE_INT) {
    int64_t i = 0;
    Check(mgp_value_get_int(value, &i));
    return static_cast<double>(i);
  }
  return kDefaultWeight;
}

// weight_property == nullptr: an unweighted view (view.weight stays empty)
WeightedView PullWeightedView(mgp_graph *graph, mgp_memory *memory, const char *weight_property) {
  WeightedView view;
  std::size_t approx_edges = 0;
  Check(mgp_graph_approximate_edge_count(graph, &approx_edges));
  std::vector<int64_t> from_gid, to_gid, seen;
  from_gid.reserve(approx_edges);
  to_gid.reserve(approx_edges);
  if (weight_property) view.weight.reserve(approx_edges);
  {
    VerticesIt vertices(graph, memory);
    std::size_t visited = 0;
    for (mgp_vertex *source = vertices.Get(); source != nullptr; source = vertices.Next(), ++visited) {
      mgp_vertex_id source_id{};
      Check(mgp_vertex_get_id(source, &source_id));
      seen.push_back(source_id.as_int);
      OutEdgesIt edges(source, memory);
      for (mgp_edge *edge = edges.Get(); edge != nullptr; edge = edges.Next()) {
        mgp_vertex *destination = nullptr;
        Check(mgp_edge_get_to(edge, &destination));
        mgp_vertex_id destination_id{};
        Check(mgp_vertex_get_id(destination, &destination_id));
        from_gid.push_back(source_id.as_int);
        to_gid.push_back(destination_id.as_int);
        if (weight_property) view.weight.push_back(EdgeWeight(edge, weight_property, memory));
      }
      if ((visited & 0xFFF) == 0 && MustAbort(graph)) throw ModuleError("procedure aborted by the host");
    }
  }
  std::sort(seen.begin(), seen.end());
  // keep the edges whose endpoints both are vertices of the view (mg_graph.hpp:213-217), then only the vertices in an edge
  std::vector<char> keep(from_gid.size(), 0);
  for (std::size_t e = 0; e < from_gid.size(); ++e)
    keep[e] = std::binary_search(seen.begin(), seen.end(), from_gid[e]) && std::binary_search(seen.begin(), seen.end(), to_gid[e]);
  for (std::size_t e = 0; e < from_gid.size(); ++e)
    if (keep[e]) {
      view.gid_of_dense.push_back(from_gid[e]);
      view.gid_of_dense.push_back(to_gid[e]);
    }
  std::sort(view.gid_of_dense.begin(), view.gid_of_dense.end());
  view.gid_of_dense.erase(std::unique(view.gid_of_dense.begin(), view.gid_of_dense.end()), view.gid_of_dense.end());
  if (view.gid_of_dense.size() >= 0xFFFFFFFEull) throw ModuleError("graph has more than 2^32 - 2 vertices");
  auto dense_of = [&view](int64_t gid) {
    return static_cast<uint32_t>(std::lower_bound(view.gid_of_dense.begin(), view.gid_of_dense.end(), gid) - view.gid_of_dense.begin());
  };
  std::size_t kept = 0;
  for (std::size_t e = 0; e < from_gid.size(); ++e)
    if (keep[e]) {
      view.from.push_back(dense_of(from_gid[e]));
      view.to.push_back(dense_of(to_gid[e]));
      if (weight_property) view.weight[kept] = view.weight[e];
      ++kept;
    }
  if (weight_property) view.weight.resize(kept);
  return view;
}

// cugraph.hits.get: the directed view without weights; rows only for vertices in an edge, in ascending gid
void HitsProcedure(mgp_list *args, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  mgp_value *arg = nullptr;
  int64_t max_iterations = 0;
  double tolerance = 0.0;
  int normalized = 0;
  Check(mgp_list_at(args, 0, &arg));
  Check(mgp_value_get_int(arg, &max_iterations));
  Check(mgp_list_at(args, 1, &arg));
  Check(mgp_value_get_double(arg, &tolerance));
  Check(mgp_list_at(args, 2, &arg));
  Check(mgp_value_get_bool(arg, &normalized));

  const WeightedView view = PullWeightedView(graph, memory, nullptr);
  const uint64_t n = view.gid_of_dense.size();
  if (n == 0) return;  // mg_graph->Empty(), or no edges at all: cuGraph has no vertex to score

  mgb200_hits_params params{};
  params.max_iterations = static_cast<uint64_t>(max_iterations);  // the reference's static_cast<size_t>
  params.tolerance = tolerance;
  params.normalized = normalized;
  std::vector<double> hubs(n), authorities(n);
  {
    HitsGraph dg;
    CheckDevice(mgb200_hits_graph_create_host_u32(DeviceFromEnv(), n, view.from.size(), view.from.data(), view.to.data(),
                                                  &dg.h));
    mgb200_hits_stats stats{};
    CheckDevice(mgb200_hits_run(dg.h, &params, hubs.data(), authorities.data(), &stats));
  }

  if (mgp_result_reserve != nullptr) (void)mgp_result_reserve(result, n);
  for (uint64_t dense = 0; dense < n; ++dense)
    EmitNodeRow(graph, result, memory, view.gid_of_dense[dense], kFieldHubs, hubs[dense], kFieldAuthorities,
                authorities[dense]);
}

void Procedure(mgp_list *args, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  if (MGB200_CUGRAPH_HITS) {
    HitsProcedure(args, graph, result, memory);
    return;
  }
  std::size_t next = 0;
  mgp_value *arg = nullptr;
  std::vector<int64_t> seed_gid;
  std::vector<double> seed_value;
  if (MGB200_CUGRAPH_PERSONALIZED) {
    mgp_list *vertices = nullptr, *values = nullptr;
    Check(mgp_list_at(args, next++, &arg));
    Check(mgp_value_get_list(arg, &vertices));
    Check(mgp_list_at(args, next++, &arg));
    Check(mgp_value_get_list(arg, &values));
    std::size_t n_seeds = 0, n_values = 0;
    Check(mgp_list_size(vertices, &n_seeds));
    Check(mgp_list_size(values, &n_values));
    if (n_seeds != n_values)
      throw ModuleError("personalization_vertices and personalization_values must have the same length.");
    if (n_seeds == 0) return;
    for (std::size_t i = 0; i < n_seeds; ++i) {
      mgp_value *item = nullptr;
      mgp_vertex *vertex = nullptr;
      Check(mgp_list_at(vertices, i, &item));
      Check(mgp_value_get_vertex(item, &vertex));
      mgp_vertex_id id{};
      Check(mgp_vertex_get_id(vertex, &id));
      double value = 0.0;
      Check(mgp_list_at(values, i, &item));
      Check(mgp_value_get_double(item, &value));
      seed_gid.push_back(id.as_int);
      seed_value.push_back(value);
    }
  }
  int64_t max_iterations = 0;
  double damping_factor = 0.0, stop_epsilon = 0.0;
  const char *weight_property = nullptr;
  Check(mgp_list_at(args, next++, &arg));
  Check(mgp_value_get_int(arg, &max_iterations));
  Check(mgp_list_at(args, next++, &arg));
  Check(mgp_value_get_double(arg, &damping_factor));
  Check(mgp_list_at(args, next++, &arg));
  Check(mgp_value_get_double(arg, &stop_epsilon));
  Check(mgp_list_at(args, next++, &arg));
  Check(mgp_value_get_string(arg, &weight_property));

  const WeightedView view = PullWeightedView(graph, memory, weight_property);
  const uint64_t n = view.gid_of_dense.size();
  if (n == 0) return;  // mg_graph->Empty(), or no edges at all: cuGraph has no vertex to rank

  std::vector<uint64_t> seeds;
  std::vector<double> values;
  if (MGB200_CUGRAPH_PERSONALIZED) {
    for (std::size_t i = 0; i < seed_gid.size(); ++i) {
      const auto it = std::lower_bound(view.gid_of_dense.begin(), view.gid_of_dense.end(), seed_gid[i]);
      if (it == view.gid_of_dense.end() || *it != seed_gid[i]) continue;  // isolated seed: skipped (:116-119)
      seeds.push_back(static_cast<uint64_t>(it - view.gid_of_dense.begin()));
      values.push_back(seed_value[i]);
    }
    if (seeds.empty()) return;  // :123
  }

  mgb200_cugraph_params params{};
  params.max_iterations = static_cast<uint64_t>(max_iterations);
  params.damping_factor = damping_factor;
  params.stop_epsilon = stop_epsilon;
  params.n_personalization = seeds.size();
  params.personalization_vertices = seeds.data();
  params.personalization_values = values.data();
  std::vector<double> pageranks(n);
  {
    DeviceGraph dg;
    CheckDevice(mgb200_graph_create_host_weighted_u32(DeviceFromEnv(), n, view.from.size(), view.from.data(),
                                                      view.to.data(), view.weight.data(), &dg.h));
    mgb200_cugraph_stats stats{};
    CheckDevice(mgb200_cugraph_pagerank_run(dg.h, &params, pageranks.data(), &stats));
  }

  if (mgp_result_reserve != nullptr) (void)mgp_result_reserve(result, n);
  for (uint64_t dense = 0; dense < n; ++dense)
    EmitNodeRow(graph, result, memory, view.gid_of_dense[dense], kFieldPageRank, pageranks[dense]);
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) int mgp_init_module(struct mgp_module *module, struct mgp_memory *memory) {
  OwnedValue max_iterations, damping_factor, stop_epsilon, weight_property;
  try {
    mgp_proc *proc = nullptr;
    Check(mgp_module_add_read_procedure(module, kProcedureGet, Guarded<Procedure>, &proc));
    if (MGB200_CUGRAPH_HITS) {  // registration as in hits.cu's mgp_init_module
      OwnedValue tolerance, normalized;
      mgp_type *type_int = nullptr, *type_float = nullptr, *type_bool = nullptr, *type_node = nullptr;
      Check(mgp_type_int(&type_int));
      Check(mgp_type_float(&type_float));
      Check(mgp_type_bool(&type_bool));
      Check(mgp_type_node(&type_node));
      Check(mgp_value_make_int(100, memory, &max_iterations.v));
      Check(mgp_value_make_double(1e-5, memory, &tolerance.v));
      Check(mgp_value_make_bool(1, memory, &normalized.v));
      Check(mgp_proc_add_opt_arg(proc, "max_iterations", type_int, max_iterations.v));
      Check(mgp_proc_add_opt_arg(proc, "tolerance", type_float, tolerance.v));
      Check(mgp_proc_add_opt_arg(proc, "normalized", type_bool, normalized.v));
      Check(mgp_proc_add_result(proc, kFieldNode, type_node));
      Check(mgp_proc_add_result(proc, kFieldHubs, type_float));
      Check(mgp_proc_add_result(proc, kFieldAuthorities, type_float));
      return 0;
    }
    mgp_type *type_int = nullptr, *type_float = nullptr, *type_node = nullptr, *type_string = nullptr;
    Check(mgp_type_int(&type_int));
    Check(mgp_type_float(&type_float));
    Check(mgp_type_node(&type_node));
    Check(mgp_type_string(&type_string));
    Check(mgp_value_make_int(100, memory, &max_iterations.v));
    Check(mgp_value_make_double(0.85, memory, &damping_factor.v));
    Check(mgp_value_make_double(1e-5, memory, &stop_epsilon.v));
    Check(mgp_value_make_string("weight", memory, &weight_property.v));
    if (MGB200_CUGRAPH_PERSONALIZED) {
      mgp_type *list_node = nullptr, *list_float = nullptr;
      Check(mgp_type_list(type_node, &list_node));
      Check(mgp_type_list(type_float, &list_float));
      Check(mgp_proc_add_arg(proc, "personalization_vertices", list_node));
      Check(mgp_proc_add_arg(proc, "personalization_values", list_float));
    }
    Check(mgp_proc_add_opt_arg(proc, "max_iterations", type_int, max_iterations.v));
    Check(mgp_proc_add_opt_arg(proc, "damping_factor", type_float, damping_factor.v));
    Check(mgp_proc_add_opt_arg(proc, "stop_epsilon", type_float, stop_epsilon.v));
    Check(mgp_proc_add_opt_arg(proc, "weight_property", type_string, weight_property.v));
    Check(mgp_proc_add_result(proc, kFieldNode, type_node));
    Check(mgp_proc_add_result(proc, kFieldPageRank, type_float));
  } catch (const std::exception &) {
    return 1;
  }
  return 0;
}

__attribute__((visibility("default"))) int mgp_shutdown_module(void) { return 0; }

}  // extern "C"

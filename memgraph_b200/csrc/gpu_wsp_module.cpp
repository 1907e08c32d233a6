// memgraph_b200/csrc/gpu_wsp_module.cpp -- query module `gpu_wsp`: the engine's weighted shortest path expansion as a
// procedure.
//
// In the reference, `MATCH (a)-[*WSHORTEST ..u (e, n | e.w) total_weight]->(b)` is an engine operator
// (ExpandWeightedShortestPathCursor, src/query/plan/operator.cpp:2917-3267) with no plugin boundary, so there is nothing
// to drop in for; this module exposes the same arithmetic behind the query-module ABI instead:
//
//   CALL gpu_wsp.distances(source, weight_property = "weight", direction = 0, upper_bound = -1)
//   YIELD node, total_weight, hops
//
//   source           NODE     the vertex the expansion starts from (never produced itself, :3135)
//   weight_property  STRING   the edge property that is the weight, (e, n | e.<weight_property>)
//   direction        INTEGER  0 = OUT, 1 = IN, 2 = BOTH                      (EdgeAtom::Direction)
//   upper_bound      INTEGER  maximum path length, -1 = unbounded (the default); any other value below 1 raises the
//                             engine's "Maximum depth in weighted shortest path expansion must be at least 1." (:3116)
//   -> one row per vertex the cursor would produce, in dense (vertex iteration) order:
//      total_weight  FLOAT    the cursor's total, bit for bit.  INTEGER weights are converted to double, so totals
//                             equal the engine's integer sums while every partial sum stays below 2^53
//      hops          INTEGER  the fewest edges among the paths the cursor can return for the vertex (include/mgb200_bfs.h);
//                             the engine's size(le) whenever the shortest path is unique
//
// Weights are checked as the engine checks them: only the edges it evaluates (walked-direction edges of the vertices
// it expands).  If one is bad, the error is the engine's text for that edge -- the one with the smallest position in
// the pulled edge list, where the engine would quote whichever it met first:
//   not a number    "Weight must be numeric or a Duration, got <type>."  (TypedValue::Type names, typed_value.cpp)
//   negative        "Weight must be non-negative, got <value>."          (fmt's shortest form of the double)
//   absent (null)   "All weights should be of the same type, ..."        (the engine's text for a null weight after the
//                                                                         first hop; a null first hop is refused too)
//   NaN             "Weight must not be NaN."                             (the engine would order NaN totals arbitrarily)
//   Duration        "Duration weights are not supported by gpu_wsp."
// Not expressible here (the engine evaluates them): filter lambdas, edge-type filters, weight expressions over vertices
// or anything but one edge property, Duration weights, the existing-target (s-t) mode, and the edge list itself.
#include <algorithm>
#include <charconv>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <limits>
#include <string>
#include <vector>

#include "mgb200_bfs.h"
#include "mgb200_pagerank.h"
#include "mgp_module_common.hpp"

using namespace mgb200_module;

namespace {

constexpr const char *kFieldTotalWeight = "total_weight";
constexpr const char *kFieldHops = "hops";
constexpr int64_t kUnbounded = std::numeric_limits<int64_t>::max();

// One pulled edge's property, as read from the host.
struct EdgeWeight {
  enum Kind : uint8_t { kNumber, kAbsent, kNotNumeric, kNegative, kNan, kDuration } kind = kNumber;
  mgp_value_type type = mgp_value_type::MGP_VALUE_TYPE_NULL;
  double value = 0.0;
};

const char *TypeName(mgp_value_type type) {  // TypedValue::Type's operator<< (src/query/typed_value.cpp:1012-1055)
  switch (type) {
    case mgp_value_type::MGP_VALUE_TYPE_NULL: return "null";
    case mgp_value_type::MGP_VALUE_TYPE_BOOL: return "bool";
    case mgp_value_type::MGP_VALUE_TYPE_INT: return "int";
    case mgp_value_type::MGP_VALUE_TYPE_DOUBLE: return "double";
    case mgp_value_type::MGP_VALUE_TYPE_STRING: return "string";
    case mgp_value_type::MGP_VALUE_TYPE_LIST: return "list";
    case mgp_value_type::MGP_VALUE_TYPE_MAP: return "map";
    case mgp_value_type::MGP_VALUE_TYPE_VERTEX: return "vertex";
    case mgp_value_type::MGP_VALUE_TYPE_EDGE: return "edge";
    case mgp_value_type::MGP_VALUE_TYPE_PATH: return "path";
    case mgp_value_type::MGP_VALUE_TYPE_DATE: return "date";
    case mgp_value_type::MGP_VALUE_TYPE_LOCAL_TIME: return "local_time";
    case mgp_value_type::MGP_VALUE_TYPE_LOCAL_DATE_TIME: return "local_date_time";
    case mgp_value_type::MGP_VALUE_TYPE_DURATION: return "duration";
    case mgp_value_type::MGP_VALUE_TYPE_ZONED_DATE_TIME: return "zoned_date_time";
    case mgp_value_type::MGP_VALUE_TYPE_POINT_2D:
    case mgp_value_type::MGP_VALUE_TYPE_POINT_3D: return "point";
    case mgp_value_type::MGP_VALUE_TYPE_ENUM: return "enum";
  }
  return "unknown";
}

// fmt's "{}" for a double: the shortest round-trip digits, fixed notation for decimal exponents in [-4, 16), else
// d[.ddd]e[+-]XX (fmt's general-format bounds, the same as Python's repr).
std::string FormatDouble(double x) {
  if (std::isnan(x)) return "nan";
  if (std::isinf(x)) return x < 0 ? "-inf" : "inf";
  char buf[64];
  const auto r = std::to_chars(buf, buf + sizeof buf, x, std::chars_format::scientific);
  const std::string sci(buf, r.ptr);
  const size_t e_at = sci.find('e');
  const bool negative = sci[0] == '-';
  std::string digits;
  for (size_t i = negative ? 1 : 0; i < e_at; ++i)
    if (sci[i] != '.') digits += sci[i];
  const int exp = std::atoi(sci.c_str() + e_at + 1);
  std::string out = negative ? "-" : "";
  if (exp < -4 || exp >= 16) {
    out += digits.substr(0, 1);
    if (digits.size() > 1) out += "." + digits.substr(1);
    char e[8];
    std::snprintf(e, sizeof e, "e%c%02d", exp < 0 ? '-' : '+', std::abs(exp));
    return out + e;
  }
  if (exp < 0) return out + "0." + std::string(static_cast<size_t>(-exp - 1), '0') + digits;
  if (digits.size() <= static_cast<size_t>(exp) + 1)
    return out + digits + std::string(static_cast<size_t>(exp) + 1 - digits.size(), '0');
  return out + digits.substr(0, static_cast<size_t>(exp) + 1) + "." + digits.substr(static_cast<size_t>(exp) + 1);
}

std::string WeightError(const EdgeWeight &w) {
  switch (w.kind) {
    case EdgeWeight::kNotNumeric:
      return std::string("Weight must be numeric or a Duration, got ") + TypeName(w.type) + ".";
    case EdgeWeight::kNegative: return "Weight must be non-negative, got " + FormatDouble(w.value) + ".";
    case EdgeWeight::kAbsent:
      return "All weights should be of the same type, either numeric or a Duration. Please update the weight "
             "expression or the filter expression. For more details, visit https://memgr.ph/wsp.";
    case EdgeWeight::kNan: return "Weight must not be NaN.";
    case EdgeWeight::kDuration: return "Duration weights are not supported by gpu_wsp.";
    default: return "invalid weight";
  }
}

struct ReadWeight {
  const char *property;
  mgp_memory *memory;
  EdgeWeight operator()(mgp_edge *edge) const {
    mgp_value *value = nullptr;
    Check(mgp_edge_get_property(edge, property, memory, &value));
    OwnedValue owned;
    owned.v = value;
    EdgeWeight w;
    Check(mgp_value_get_type(value, &w.type));
    if (w.type == mgp_value_type::MGP_VALUE_TYPE_DOUBLE) {
      Check(mgp_value_get_double(value, &w.value));
    } else if (w.type == mgp_value_type::MGP_VALUE_TYPE_INT) {
      int64_t i = 0;
      Check(mgp_value_get_int(value, &i));
      w.value = static_cast<double>(i);
    } else {
      w.kind = w.type == mgp_value_type::MGP_VALUE_TYPE_NULL       ? EdgeWeight::kAbsent
               : w.type == mgp_value_type::MGP_VALUE_TYPE_DURATION ? EdgeWeight::kDuration
                                                                   : EdgeWeight::kNotNumeric;
      return w;
    }
    if (std::isnan(w.value)) w.kind = EdgeWeight::kNan;
    else if (w.value < 0.0) w.kind = EdgeWeight::kNegative;
    return w;
  }
};

void Distances(mgp_list *args, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  mgp_value *arg = nullptr;
  mgp_vertex *source = nullptr;
  const char *property = nullptr;
  int64_t direction = 0, upper = -1;
  Check(mgp_list_at(args, 0, &arg));
  Check(mgp_value_get_vertex(arg, &source));
  Check(mgp_list_at(args, 1, &arg));
  Check(mgp_value_get_string(arg, &property));
  Check(mgp_list_at(args, 2, &arg));
  Check(mgp_value_get_int(arg, &direction));
  Check(mgp_list_at(args, 3, &arg));
  Check(mgp_value_get_int(arg, &upper));
  if (direction < MGB200_BFS_OUT || direction > MGB200_BFS_BOTH)
    throw ModuleError("direction must be 0 (OUT), 1 (IN) or 2 (BOTH)");
  if (upper == -1) upper = kUnbounded;
  if (upper < 1) throw ModuleError("Maximum depth in weighted shortest path expansion must be at least 1.");
  mgp_vertex_id source_id{};
  Check(mgp_vertex_get_id(source, &source_id));

  // edges to vertices the iterator never showed are dropped, as gpu_bfs does: a fabricated edge would change totals
  std::vector<EdgeWeight> weights;
  const HostGraph hg = PullGraph(graph, memory, UnknownGid::kUnknownDropped, ReadWeight{property, memory}, &weights);
  const uint64_t n = hg.gid_of_dense.size(), m = hg.from.size();
  uint64_t source_dense = n;
  if (!hg.dense_of_gid.Find(source_id.as_int, &source_dense)) throw ModuleError("Invalid ID!");

  std::vector<double> w(m);
  for (uint64_t e = 0; e < m; ++e)
    w[e] = weights[e].kind == EdgeWeight::kNumber ? weights[e].value : std::numeric_limits<double>::quiet_NaN();
  std::vector<double> dist(n);
  std::vector<int32_t> hops(n);
  {
    const BfsDeviceGraph dg(hg);
    mgb200_wsp_stats stats{};
    int rc = mgb200_bfs_graph_set_weights(dg.graph.h, m, dg.from.data(), dg.to.data(), w.data());
    if (rc == MGB200_OK)
      rc = mgb200_wsp_run(dg.graph.h, source_dense, static_cast<int>(direction), upper, MustAbortPoll, graph,
                          dist.data(), hops.data(), &stats);
    if (rc == MGB200_ERR_INVALID_WEIGHT) throw ModuleError(WeightError(weights[stats.invalid_edge]));
    CheckDevice(rc);
  }

  for (uint64_t v = 0; v < n; ++v)
    if (hops[v] >= 0)
      EmitNodeRow(graph, result, memory, hg.gid_of_dense[v], kFieldTotalWeight, dist[v], kFieldHops, hops[v]);
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) int mgp_init_module(struct mgp_module *module, struct mgp_memory *memory) {
  OwnedValue weight_property, direction, upper;
  try {
    mgp_proc *proc = nullptr;
    Check(mgp_module_add_read_procedure(module, "distances", Guarded<Distances>, &proc));
    mgp_type *type_int = nullptr, *type_float = nullptr, *type_node = nullptr, *type_string = nullptr;
    Check(mgp_type_int(&type_int));
    Check(mgp_type_float(&type_float));
    Check(mgp_type_node(&type_node));
    Check(mgp_type_string(&type_string));
    Check(mgp_proc_add_arg(proc, "source", type_node));
    Check(mgp_value_make_string("weight", memory, &weight_property.v));
    Check(mgp_value_make_int(0, memory, &direction.v));
    Check(mgp_value_make_int(-1, memory, &upper.v));
    Check(mgp_proc_add_opt_arg(proc, "weight_property", type_string, weight_property.v));
    Check(mgp_proc_add_opt_arg(proc, "direction", type_int, direction.v));
    Check(mgp_proc_add_opt_arg(proc, "upper_bound", type_int, upper.v));
    Check(mgp_proc_add_result(proc, kFieldNode, type_node));
    Check(mgp_proc_add_result(proc, kFieldTotalWeight, type_float));
    Check(mgp_proc_add_result(proc, kFieldHops, type_int));
  } catch (...) {
    return 1;
  }
  return 0;
}

__attribute__((visibility("default"))) int mgp_shutdown_module(void) { return 0; }

}  // extern "C"

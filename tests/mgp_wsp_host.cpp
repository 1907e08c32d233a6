// tests/mgp_wsp_host.cpp -- TEST INFRASTRUCTURE: the fake mgp host of tests/mgp_fake_host.cpp, unchanged, plus what the
// gpu_wsp module's tests need beyond it:
//   * fh_wsp_call: CallCustomProcedure with typed arguments ('v' NODE by gid, 's' STRING, 'i' INTEGER, 'd' FLOAT) under
//     the base host's strict type check, returning the `node` column, one FLOAT column and one INTEGER column by name
//     (fh_call copies one value column only);
//   * tagged edge properties: an edge whose numeric property (fh_graph_set_edge_property) holds one of the NaN bit
//     patterns below hands out the STRING "not a number" (kStringWeightBits), a DOUBLE NaN (kNanWeightBits) or a
//     DURATION (kDurationWeightBits) instead, so every weight error can be reached.  Every other NaN still means "the
//     edge lacks the property".  The base host has no DURATION kind: such a value is a Null whose string is
//     "duration", and mgp_value_get_type reports it as MGP_VALUE_TYPE_DURATION.
// It builds its own library (memgraph_b200/_build/libmgp_wsp_host.so); like the other hosts it defines every mgp_*
// symbol, so one process loads only one host (tests/test_wsp_module.py runs each call in a child interpreter).
#define mgp_edge_get_property fh_base_edge_get_property
#define mgp_value_get_type fh_base_value_get_type
#include "mgp_fake_host.cpp"
#undef mgp_edge_get_property
#undef mgp_value_get_type

constexpr uint64_t kStringWeightBits = 0x7FF8000053545200ull;    // a quiet NaN with the payload "STR"
constexpr uint64_t kNanWeightBits = 0x7FF800004E414E00ull;       // "NAN"
constexpr uint64_t kDurationWeightBits = 0x7FF8000044555200ull;  // "DUR"
constexpr const char *kDurationMarker = "duration";

struct FhWspResult {
  std::string error;  // empty = success
  std::vector<int64_t> nodes;
  std::vector<double> floats;
  std::vector<int64_t> ints;
};

extern "C" {

mgp_error mgp_value_get_type(mgp_value *val, mgp_value_type *result) {
  if (val->kind == ValueKind::Null && val->s == kDurationMarker) {
    *result = mgp_value_type::MGP_VALUE_TYPE_DURATION;
    return OK;
  }
  return fh_base_value_get_type(val, result);
}

mgp_error mgp_edge_get_property(mgp_edge *e, const char *property_name, mgp_memory *memory, mgp_value **result) {
  uint64_t bits = 0;
  std::memcpy(&bits, &e->prop, sizeof bits);
  const FakeGraphData *d = e->from.graph->data;
  const bool tagged = bits == kStringWeightBits || bits == kNanWeightBits || bits == kDurationWeightBits;
  if (!tagged || !property_name || d->prop_name != property_name)
    return fh_base_edge_get_property(e, property_name, memory, result);
  if (memory) memory->allocations++;
  auto *x = new (std::nothrow) mgp_value();
  if (!x) return mgp_error::MGP_ERROR_UNABLE_TO_ALLOCATE;
  if (bits == kStringWeightBits) {
    x->kind = ValueKind::String;
    x->s = "not a number";
  } else if (bits == kNanWeightBits) {
    x->kind = ValueKind::Double;
    x->d = std::numeric_limits<double>::quiet_NaN();
  } else {
    x->s = kDurationMarker;  // kind stays Null
  }
  x->counted = true;
  g_live_objects++;
  *result = x;
  return OK;
}

// kinds[i]: 'v' NODE (gid in ivals), 's' STRING (svals[i]), 'i' INTEGER (ivals), 'd' FLOAT (dvals); missing optional
// arguments take their defaults.
void *fh_wsp_call(void *module, const char *proc_name, void *graph_data, int n_args, const char *kinds,
                  const int64_t *ivals, const double *dvals, const char *const *svals, const char *float_column,
                  const char *int_column) {
  auto *m = static_cast<FhModule *>(module);
  auto *res_out = new FhWspResult();
  auto it = m->registry.procs.find(proc_name);
  if (it == m->registry.procs.end()) {
    res_out->error = "There is no procedure named '" + m->name + "." + proc_name + "'.";
    return res_out;
  }
  mgp_proc &proc = it->second;
  const std::string fq = m->name + "." + proc.name;
  size_t n_required = 0;
  for (auto &a : proc.opt_args) n_required += a.required;
  if (n_args < 0 || static_cast<size_t>(n_args) > proc.opt_args.size() || static_cast<size_t>(n_args) < n_required) {
    res_out->error = "'" + fq + "' requires between " + std::to_string(n_required) + " and " +
                     std::to_string(proc.opt_args.size()) + " arguments.";
    return res_out;
  }
  mgp_graph graph{static_cast<FakeGraphData *>(graph_data)};
  std::vector<std::unique_ptr<mgp_vertex>> arg_vertices;
  mgp_list args;
  for (size_t i = 0; i < proc.opt_args.size(); ++i) {
    mgp_value v;
    if (i < static_cast<size_t>(n_args)) {
      const char k = kinds[i];
      const ValueKind given = k == 'i' ? ValueKind::Int : k == 'v' ? ValueKind::Vertex : k == 's' ? ValueKind::String
                                                                                                   : ValueKind::Double;
      if (given != proc.opt_args[i].type->kind) {  // strict: an integer literal does not satisfy FLOAT
        res_out->error = "'" + fq + "' argument named '" + proc.opt_args[i].name + "' at position " +
                         std::to_string(i) + " must be of type " + proc.opt_args[i].type->name + ".";
        return res_out;
      }
      v.kind = given;
      v.i = ivals[i];
      v.d = dvals[i];
      if (given == ValueKind::String) v.s = (svals && svals[i]) ? svals[i] : "";
      if (given == ValueKind::Vertex) {
        auto found = graph.data->index_of.find(ivals[i]);
        if (found == graph.data->index_of.end()) {
          res_out->error = "'" + fq + "': no vertex with the given id";
          return res_out;
        }
        arg_vertices.push_back(std::make_unique<mgp_vertex>(mgp_vertex{&graph, found->second, false}));
        v.vertex = arg_vertices.back().get();
      }
    } else {
      v = proc.opt_args[i].default_value;
    }
    args.items.push_back(v);
  }
  mgp_result result;
  result.proc = &proc;
  mgp_memory memory;
  proc.cb(&args, &graph, &result, &memory);
  if (result.has_error) {
    res_out->error = fq + ": " + result.error;
    return res_out;
  }
  for (auto &row : result.rows) {
    int64_t node = -1, iv = 0;
    double fv = 0.0;
    for (size_t f = 0; f < proc.results.size(); ++f) {
      if (proc.results[f].first == "node") node = row->fields[f].i;
      if (proc.results[f].first == float_column && row->fields[f].kind == ValueKind::Double) fv = row->fields[f].d;
      if (proc.results[f].first == int_column && row->fields[f].kind == ValueKind::Int) iv = row->fields[f].i;
    }
    res_out->nodes.push_back(node);
    res_out->floats.push_back(fv);
    res_out->ints.push_back(iv);
  }
  return res_out;
}

const char *fh_wsp_result_error(void *result) {
  auto *r = static_cast<FhWspResult *>(result);
  return r->error.empty() ? nullptr : r->error.c_str();
}
uint64_t fh_wsp_result_rows(void *result) { return static_cast<FhWspResult *>(result)->nodes.size(); }
void fh_wsp_result_copy(void *result, int64_t *nodes, double *floats, int64_t *ints) {
  auto *r = static_cast<FhWspResult *>(result);
  if (!r->nodes.empty()) {
    std::memcpy(nodes, r->nodes.data(), r->nodes.size() * sizeof(int64_t));
    std::memcpy(floats, r->floats.data(), r->floats.size() * sizeof(double));
    std::memcpy(ints, r->ints.data(), r->ints.size() * sizeof(int64_t));
  }
}
void fh_wsp_result_destroy(void *result) { delete static_cast<FhWspResult *>(result); }

}  // extern "C"

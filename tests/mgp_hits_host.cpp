// tests/mgp_hits_host.cpp -- TEST INFRASTRUCTURE: the BOOLEAN / edge-id host of tests/mgp_bc_host.cpp, unchanged, plus
// one call entry for procedures whose rows carry a node and two FLOAT columns picked by name (fh_bc_call copies one
// FLOAT column, whichever comes last).  Arguments are typed as in fh_bc_call: 'i' INTEGER, 'd' FLOAT, 'b' BOOLEAN, under
// the same strict type check; missing optional arguments take their defaults.  It builds its own library
// (memgraph_b200/_build/libmgp_hits_host.so); like the other hosts it defines every mgp_* symbol, so one process loads
// only one host (tests/test_hits_module.py runs each call in a child interpreter).
#include "mgp_bc_host.cpp"

struct FhColumnsResult {
  std::string error;  // empty = success
  std::vector<int64_t> nodes;
  std::vector<double> first, second;
};

extern "C" {

void *fh_columns_call(void *module, const char *proc_name, void *graph_data, int n_args, const char *kinds,
                      const int64_t *ivals, const double *dvals, const char *first, const char *second) {
  auto *m = static_cast<FhModule *>(module);
  auto *res_out = new FhColumnsResult();
  auto it = m->registry.procs.find(proc_name);
  if (it == m->registry.procs.end()) {
    res_out->error = "There is no procedure named '" + m->name + "." + proc_name + "'.";
    return res_out;
  }
  mgp_proc &proc = it->second;
  const std::string fq = m->name + "." + proc.name;
  if (n_args < 0 || static_cast<size_t>(n_args) > proc.opt_args.size()) {
    res_out->error = "'" + fq + "' requires between 0 and " + std::to_string(proc.opt_args.size()) + " arguments.";
    return res_out;
  }
  mgp_list args;
  for (size_t i = 0; i < proc.opt_args.size(); ++i) {
    mgp_value v = proc.opt_args[i].default_value;
    if (i < static_cast<size_t>(n_args)) {
      const mgp_type *want = proc.opt_args[i].type;
      const bool ok = want == &g_type_bool ? kinds[i] == 'b'
                                           : (kinds[i] == 'i' && want->kind == ValueKind::Int) ||
                                                 (kinds[i] == 'd' && want->kind == ValueKind::Double);
      if (!ok) {
        res_out->error = "'" + fq + "' argument named '" + proc.opt_args[i].name + "' at position " +
                         std::to_string(i) + " must be of type " + want->name + ".";
        return res_out;
      }
      v = mgp_value{};
      v.kind = want->kind;
      v.i = kinds[i] == 'b' ? (ivals[i] != 0) : ivals[i];
      v.d = dvals[i];
    }
    args.items.push_back(v);
  }
  mgp_graph graph{static_cast<FakeGraphData *>(graph_data)};
  mgp_result result;
  result.proc = &proc;
  mgp_memory memory;
  proc.cb(&args, &graph, &result, &memory);
  if (result.has_error) {
    res_out->error = fq + ": " + result.error;
    return res_out;
  }
  for (auto &row : result.rows) {
    int64_t node = -1;
    double a = 0.0, b = 0.0;
    for (size_t f = 0; f < proc.results.size(); ++f) {
      const auto &[name, type] = proc.results[f];
      if (name == "node") node = row->fields[f].i;
      if (type->kind != ValueKind::Double) continue;
      if (name == first) a = row->fields[f].d;
      if (name == second) b = row->fields[f].d;
    }
    res_out->nodes.push_back(node);
    res_out->first.push_back(a);
    res_out->second.push_back(b);
  }
  return res_out;
}

const char *fh_columns_result_error(void *result) {
  auto *r = static_cast<FhColumnsResult *>(result);
  return r->error.empty() ? nullptr : r->error.c_str();
}
uint64_t fh_columns_result_rows(void *result) { return static_cast<FhColumnsResult *>(result)->nodes.size(); }
void fh_columns_result_copy(void *result, int64_t *nodes, double *first, double *second) {
  auto *r = static_cast<FhColumnsResult *>(result);
  if (!r->nodes.empty()) {
    std::memcpy(nodes, r->nodes.data(), r->nodes.size() * sizeof(int64_t));
    std::memcpy(first, r->first.data(), r->first.size() * sizeof(double));
    std::memcpy(second, r->second.data(), r->second.size() * sizeof(double));
  }
}
void fh_columns_result_destroy(void *result) { delete static_cast<FhColumnsResult *>(result); }

}  // extern "C"

// tests/mgp_wcc_host.cpp -- TEST INFRASTRUCTURE: the BOOLEAN / edge-id host of tests/mgp_bc_host.cpp, unchanged, plus
// one call entry for procedures whose result is a node column and an INTEGER column (fh_bc_call and fh_call copy
// FLOAT columns only).  It builds its own library (memgraph_b200/_build/libmgp_wcc_host.so); like the other hosts it
// defines every mgp_* symbol, so one process loads only one host (tests/test_wcc_module.py runs each call in a child
// interpreter).
#include "mgp_bc_host.cpp"

struct FhIntResult {
  std::string error;  // empty = success
  std::vector<int64_t> nodes;
  std::vector<int64_t> values;
};

extern "C" {

// A procedure without arguments; returns the `node` column and the INTEGER column named `column` of every row.
void *fh_int_call(void *module, const char *proc_name, void *graph_data, const char *column) {
  auto *m = static_cast<FhModule *>(module);
  auto *res_out = new FhIntResult();
  auto it = m->registry.procs.find(proc_name);
  if (it == m->registry.procs.end()) {
    res_out->error = "There is no procedure named '" + m->name + "." + proc_name + "'.";
    return res_out;
  }
  mgp_proc &proc = it->second;
  const std::string fq = m->name + "." + proc.name;
  mgp_list args;
  for (const auto &a : proc.opt_args) args.items.push_back(a.default_value);
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
    int64_t node = -1, value = 0;
    for (size_t f = 0; f < proc.results.size(); ++f) {
      if (proc.results[f].first == "node") node = row->fields[f].i;
      if (proc.results[f].first == column && proc.results[f].second->kind == ValueKind::Int) value = row->fields[f].i;
    }
    res_out->nodes.push_back(node);
    res_out->values.push_back(value);
  }
  return res_out;
}

const char *fh_int_result_error(void *result) {
  auto *r = static_cast<FhIntResult *>(result);
  return r->error.empty() ? nullptr : r->error.c_str();
}
uint64_t fh_int_result_rows(void *result) { return static_cast<FhIntResult *>(result)->nodes.size(); }
void fh_int_result_copy(void *result, int64_t *nodes, int64_t *values) {
  auto *r = static_cast<FhIntResult *>(result);
  if (!r->nodes.empty()) {
    std::memcpy(nodes, r->nodes.data(), r->nodes.size() * sizeof(int64_t));
    std::memcpy(values, r->values.data(), r->values.size() * sizeof(int64_t));
  }
}
void fh_int_result_destroy(void *result) { delete static_cast<FhIntResult *>(result); }

}  // extern "C"

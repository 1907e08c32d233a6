// tests/mgp_edge_host.cpp -- TEST INFRASTRUCTURE: the INTEGER-column host of tests/mgp_wcc_host.cpp, unchanged, plus
// one call entry for procedures whose rows are edges: an optional INTEGER column and the `node_from` / `node_to` NODE
// columns (bridges.get, biconnected_components.get).  It builds its own library
// (memgraph_b200/_build/libmgp_edge_host.so); like the other hosts it defines every mgp_* symbol, so one process loads
// only one host (tests/test_biconnectivity_modules.py runs each call in a child interpreter).
#include "mgp_wcc_host.cpp"

struct FhEdgeResult {
  std::string error;  // empty = success
  std::vector<int64_t> values, from, to;
};

extern "C" {

// A procedure without arguments; returns, per row, the INTEGER column named `column` (0 when column is null or the
// procedure has no such column) and the gids of `node_from` and `node_to`.
void *fh_edge_call(void *module, const char *proc_name, void *graph_data, const char *column) {
  auto *m = static_cast<FhModule *>(module);
  auto *res_out = new FhEdgeResult();
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
    int64_t value = 0, from = -1, to = -1;
    for (size_t f = 0; f < proc.results.size(); ++f) {
      const auto &[name, type] = proc.results[f];
      if (name == "node_from" && type->kind == ValueKind::Vertex) from = row->fields[f].i;
      if (name == "node_to" && type->kind == ValueKind::Vertex) to = row->fields[f].i;
      if (column && name == column && type->kind == ValueKind::Int) value = row->fields[f].i;
    }
    res_out->values.push_back(value);
    res_out->from.push_back(from);
    res_out->to.push_back(to);
  }
  return res_out;
}

const char *fh_edge_result_error(void *result) {
  auto *r = static_cast<FhEdgeResult *>(result);
  return r->error.empty() ? nullptr : r->error.c_str();
}
uint64_t fh_edge_result_rows(void *result) { return static_cast<FhEdgeResult *>(result)->from.size(); }
void fh_edge_result_copy(void *result, int64_t *values, int64_t *from, int64_t *to) {
  auto *r = static_cast<FhEdgeResult *>(result);
  if (!r->from.empty()) {
    std::memcpy(values, r->values.data(), r->values.size() * sizeof(int64_t));
    std::memcpy(from, r->from.data(), r->from.size() * sizeof(int64_t));
    std::memcpy(to, r->to.data(), r->to.size() * sizeof(int64_t));
  }
}
void fh_edge_result_destroy(void *result) { delete static_cast<FhEdgeResult *>(result); }

}  // extern "C"

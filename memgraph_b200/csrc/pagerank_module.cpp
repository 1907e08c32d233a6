// memgraph_b200/csrc/pagerank_module.cpp -- the drop-in `pagerank` query module (host side, C++).
//
// Replaces mage/cpp/pagerank_module/pagerank_module.cpp of the reference behind the same ABI:
//   CALL pagerank.get(max_iterations = 100, damping_factor = 0.85, stop_epsilon = 1e-5, num_of_threads = 1)
//   YIELD node, rank                                                      (reference :116-155)
// Same procedure name, argument names / types / defaults / order, result fields, one row per
// vertex in vertex-iteration order, same error texts.  What differs is where the arithmetic runs:
// the graph is pulled ONCE through the mgp_graph iterators (reference CreatePageRankGraph :18-54),
// shipped to the GPU, iterated there (include/mgb200_pagerank.h), and the ranks come back as one
// double[N] that is turned into records (reference InsertPagerankRecord :69-84).
//
// Build: memgraph_b200/build.py links this file with the CUDA objects and a static CUDA runtime into
// memgraph_b200/_build/pagerank.so, whose only undefined symbols are mgp_* (plus libc/libstdc++),
// as dlopen(RTLD_NOW | RTLD_LOCAL) in src/query/procedure/module.cpp:861 requires.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <stdexcept>
#include <mutex>
#include <string>
#include <vector>

#include "mgb200_pagerank.h"
#include "mgp_module_common.hpp"

using namespace mgb200_module;

namespace {

constexpr const char *kProcedureGet = "get";
constexpr const char *kFieldRank = "rank";
constexpr const char *kArgMaxIterations = "max_iterations";
constexpr const char *kArgDampingFactor = "damping_factor";
constexpr const char *kArgStopEpsilon = "stop_epsilon";
constexpr const char *kArgNumThreads = "num_of_threads";

struct DeviceGraphCache {
  std::mutex busy;
  mgb200_graph *graph = nullptr;
  uint64_t n = 0, m = 0, fp[2] = {0, 0}, hits = 0;
  int device = -1;
  ~DeviceGraphCache() { mgb200_graph_destroy(graph); }
};

std::vector<double> ComputeRanks(const HostGraph &hg, mgp_graph *graph, int64_t max_iterations, double damping_factor,
                                 double stop_epsilon, int64_t num_threads) {
  // pagerank.hpp:109 takes uint32_t, pagerank.cpp:195 clamps to hardware_concurrency, :63-65 rejects 0.
  const uint32_t threads = static_cast<uint32_t>(num_threads);
  if (threads == 0) throw ModuleError(MGB200_MSG_ZERO_THREADS);
  const uint64_t n = hg.gid_of_dense.size();
  std::vector<double> ranks(n);
  if (n == 0) return ranks;
  mgb200_run_params params{};
  params.max_iterations = static_cast<uint64_t>(max_iterations);  // int64 -> size_t wrap, reference :95
  params.damping_factor = damping_factor;
  params.stop_epsilon = stop_epsilon;
  params.should_abort = MustAbortPoll;  // polled between iteration batches, from this thread only
  params.abort_user = graph;
  // MGB200_GPUS=P (2..8): vertex-partition the call over GPUs 0..P-1 (device-side exchange over NVLink)
  const char *gpus_env = std::getenv("MGB200_GPUS");
  const int gpus = gpus_env ? std::atoi(gpus_env) : 1;
  if (gpus > 1) {
    uint64_t iterations = 0;
    CheckDevice(mgb200_pagerank_multi_u32(n, hg.from.size(), hg.from.data(), hg.to.data(), &params, threads,
                                          static_cast<uint32_t>(gpus), nullptr, ranks.data(), &iterations));
    return ranks;
  }
  const int device = DeviceFromEnv();
  // MGB200_GRAPH_CACHE=1: keep the device-resident graph across CALLs.  The mgp ABI has no graph version, so the key is a
  // 128-bit fingerprint of the dense COO just pulled (plus n, m, device): an unchanged graph skips the upload and the
  // device build, a changed one replaces the slot.  One slot, taken with try_lock: a concurrent second query (the module is
  // shared between sessions, src/query/plan/operator.cpp:7808-7829) simply builds its own throw-away graph.
  static DeviceGraphCache cache;
  const char *cache_env = std::getenv("MGB200_GRAPH_CACHE");
  std::unique_lock<std::mutex> slot(cache.busy, std::defer_lock);
  const bool use_cache = cache_env && cache_env[0] == '1' && slot.try_lock();
  DeviceGraph owned;  // the handle of a call that does not hand it to the cache
  mgb200_graph *dg = nullptr;
  if (use_cache) {
    uint64_t fp[2] = {0, 0};
    CheckDevice(mgb200_coo_fingerprint_u32(n, hg.from.size(), hg.from.data(), hg.to.data(), fp));
    if (cache.graph && cache.n == n && cache.m == hg.from.size() && cache.device == device && cache.fp[0] == fp[0] &&
        cache.fp[1] == fp[1]) {
      ++cache.hits;
    } else {
      mgb200_graph_destroy(cache.graph);
      cache.graph = nullptr;
      CheckDevice(mgb200_graph_create_host_u32(device, n, hg.from.size(), hg.from.data(), hg.to.data(), 0, 1, &owned.h));
      cache.graph = owned.Release();
      cache.n = n;
      cache.m = hg.from.size();
      cache.device = device;
      cache.fp[0] = fp[0];
      cache.fp[1] = fp[1];
    }
    dg = cache.graph;
  } else {
    CheckDevice(mgb200_graph_create_host_u32(device, n, hg.from.size(), hg.from.data(), hg.to.data(), 0, 1, &owned.h));
    dg = owned.h;
  }
  mgb200_run_stats stats{};
  CheckDevice(mgb200_pagerank_run(dg, &params, ranks.data(), &stats));
  return ranks;
}

// Nothing may escape the callback (reference :108-112); Guarded turns an exception into the error message, which the
// engine reports as QueryRuntimeException("pagerank.get: <msg>") (src/query/plan/operator.cpp:7929-7932).
void PagerankGet(mgp_list *args, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  mgp_value *arg = nullptr;
  int64_t max_iterations = 0, num_threads = 0;
  double damping_factor = 0.0, stop_epsilon = 0.0;
  Check(mgp_list_at(args, 0, &arg));
  Check(mgp_value_get_int(arg, &max_iterations));
  Check(mgp_list_at(args, 1, &arg));
  Check(mgp_value_get_double(arg, &damping_factor));
  Check(mgp_list_at(args, 2, &arg));
  Check(mgp_value_get_double(arg, &stop_epsilon));
  Check(mgp_list_at(args, 3, &arg));
  Check(mgp_value_get_int(arg, &num_threads));

  const HostGraph hg = PullGraph(graph, memory);
  const std::vector<double> ranks =
      ComputeRanks(hg, graph, max_iterations, damping_factor, stop_epsilon, num_threads);

  if (mgp_result_reserve != nullptr && !ranks.empty()) (void)mgp_result_reserve(result, ranks.size());
  // one (node, rank) row per vertex (reference InsertPagerankRecord :69-84)
  for (std::size_t dense = 0; dense < ranks.size(); ++dense)
    EmitNodeRow(graph, result, memory, hg.gid_of_dense[dense], kFieldRank, ranks[dense]);
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) int mgp_init_module(struct mgp_module *module, struct mgp_memory *memory) {
  OwnedValue max_iterations, damping_factor, stop_epsilon, num_threads;  // destroyed on every path (:139-152)
  try {
    mgp_proc *proc = nullptr;
    Check(mgp_module_add_read_procedure(module, kProcedureGet, Guarded<PagerankGet>, &proc));
    Check(mgp_value_make_int(100, memory, &max_iterations.v));
    Check(mgp_value_make_double(0.85, memory, &damping_factor.v));
    Check(mgp_value_make_double(1e-5, memory, &stop_epsilon.v));
    Check(mgp_value_make_int(1, memory, &num_threads.v));
    mgp_type *type_int = nullptr, *type_float = nullptr, *type_node = nullptr;
    Check(mgp_type_int(&type_int));
    Check(mgp_type_float(&type_float));
    Check(mgp_type_node(&type_node));
    Check(mgp_proc_add_opt_arg(proc, kArgMaxIterations, type_int, max_iterations.v));
    Check(mgp_proc_add_opt_arg(proc, kArgDampingFactor, type_float, damping_factor.v));
    Check(mgp_proc_add_opt_arg(proc, kArgStopEpsilon, type_float, stop_epsilon.v));
    Check(mgp_proc_add_opt_arg(proc, kArgNumThreads, type_int, num_threads.v));
    Check(mgp_proc_add_result(proc, kFieldNode, type_node));
    Check(mgp_proc_add_result(proc, kFieldRank, type_float));
  } catch (...) {
    return 1;
  }
  return 0;
}

__attribute__((visibility("default"))) int mgp_shutdown_module(void) { return 0; }

}  // extern "C"

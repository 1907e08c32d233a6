// memgraph_b200/csrc/wsp.cu -- weighted shortest paths from one source for sm_90a (include/mgb200_bfs.h).
//
// Semantics: ExpandWeightedShortestPathCursor, src/query/plan/operator.cpp:2917-3267 (restated and pinned in
// oracle/wsp_oracle.c), one source, unbound target, one numeric edge property as the weight, no filter lambda.
//
// Exactness.  Distances are the bit patterns of non-negative doubles held in uint64 (for w >= +0 the patterns order
// like the values, so atomicMin on the bits is a min on the values); kUnreached sits above +inf, so a vertex reached at
// +inf stays distinguishable.  Every addition is an explicit __dadd_rn.  Because fl(a + w) is monotone in a and never
// below a, any relaxation order converges to the least fixed point of d[v] = min_u fl(d[u] + w_uv), which is what
// the reference's Dijkstra yields; and because fl(min a_i + w) = min fl(a_i + w), a Jacobi Bellman-Ford round k gives
// exactly the minimum over walks of at most k edges.
//
// Passes.  Every pass reads only values frozen before it: the frontier carries (vertex, its distance when the pass
// started); the pass lowers dist[] with atomicMin and lists each lowered vertex once (a per-vertex pass stamp); a
// classify step then reads the lowered vertices' final values.  So the frontier of every pass is a set that does not
// depend on thread order, and two runs give the same outputs and the same counters.
//   bounded (upper_bound = u)   at most u Jacobi Bellman-Ford passes; the lowered vertices of pass k are the frontier
//                               of pass k + 1 and get hops = k, so hops ends as the round of the last strict
//                               improvement, the smallest k with d_k[v] = d_u[v]
//   unbounded                   delta-stepping with a near and a far pile (Davidson et al.): passes run while the near
//                               pile (distance below the bucket threshold T) is not empty; lowered vertices at or above
//                               T go to the far pile once per bucket (a per-vertex bucket stamp).  When the near pile is
//                               empty, T moves to the end of the bucket holding the smallest far distance and the far
//                               pile is split; an entry below the old T was already handled through the near pile.
//                               Then a level-synchronous BFS over the tight entries (d[v] == fl(d[u] + w)) gives hops.
// Work split.  A frontier vertex's list is cut into kSegEdges-entry segments and one warp walks each segment (the
// segment scan of bfs.cu), so an RMAT hub with 10^6 entries is spread over a thousand warps.
// Invalid entries (negative or NaN weights, stored as kInvalidTag | COO index) are never relaxed; the smallest index
// among the inspected ones is kept with atomicMin.  An entry is inspected exactly when the reference evaluates it: the
// walked-direction entries of every vertex it expands (every reached vertex; bounded, those reached within u - 1 hops).
#include <cub/cub.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "bfs_graph.hpp"
#include "core.hpp"
#include "mgb200_bfs.h"

namespace mgb200 {
namespace {

constexpr uint32_t kSegEdges = 1024;
constexpr uint64_t kInfBits = 0x7FF0000000000000ull;
constexpr uint64_t kUnreached = 0x7FF0000000000001ull;  // above +inf, below every NaN
constexpr uint64_t kInvalidTag = MGB200_WSP_INVALID_TAG;
constexpr uint64_t kIndexMask = (1ull << 51) - 1;

struct WAdj {  // the lists a direction walks: `a` first, then `b` (BOTH), with their weights
  const uint64_t *a_ptr;
  const uint32_t *a_adj;
  const uint64_t *a_w;
  const uint64_t *b_ptr;  // nullptr unless BOTH
  const uint32_t *b_adj;
  const uint64_t *b_w;
  __device__ __forceinline__ uint64_t degree(uint32_t u) const {
    uint64_t d = a_ptr[u + 1] - a_ptr[u];
    if (b_ptr) d += b_ptr[u + 1] - b_ptr[u];
    return d;
  }
  __device__ __forceinline__ void entry(uint32_t u, uint64_t k, uint32_t *v, uint64_t *w) const {
    const uint64_t a0 = a_ptr[u], da = a_ptr[u + 1] - a0;
    if (k < da) {
      *v = a_adj[a0 + k];
      *w = a_w[a0 + k];
    } else {
      const uint64_t i = b_ptr[u] + (k - da);
      *v = b_adj[i];
      *w = b_w[i];
    }
  }
};

struct Counters {
  unsigned long long lowered;    // vertices the pass lowered (the improved list)
  unsigned long long near;       // near-pile entries written by classify / split
  unsigned long long far;        // far-pile entries
  unsigned long long inspected;  // adjacency entries read
  unsigned long long invalid;    // smallest inspected invalid COO index (~0 = none)
  unsigned long long far_min;    // smallest far distance at or above T (~0 = none)
  unsigned long long reached;    // produced vertices
  unsigned long long max_hops;
};

__device__ __forceinline__ uint64_t add_bits(uint64_t d, uint64_t w) {
  return static_cast<uint64_t>(__double_as_longlong(__dadd_rn(__longlong_as_double(static_cast<long long>(d)),
                                                              __longlong_as_double(static_cast<long long>(w)))));
}

// Warp-aggregated append of the lanes whose `take` is set.
__device__ __forceinline__ void warp_push(bool take, uint32_t value, uint32_t *list, unsigned long long *count) {
  const unsigned ballot = __ballot_sync(kFull, take);
  if (!ballot) return;
  const int lane = threadIdx.x & 31, leader = __ffs(ballot) - 1;
  unsigned long long base = 0;
  if (lane == leader) base = atomicAdd(count, static_cast<unsigned long long>(__popc(ballot)));
  base = __shfl_sync(kFull, base, leader);
  if (take) list[base + __popc(ballot & ((1u << lane) - 1u))] = value;
}

__global__ void init_kernel(uint64_t n, uint32_t source, uint64_t *dist, int32_t *hops, uint32_t *stamp,
                            uint32_t *bucket_stamp, uint32_t *near_v, uint64_t *near_d, Counters *c) {
  for (uint64_t v = first_thread(); v < n; v += thread_count()) {
    dist[v] = v == source ? 0ull : kUnreached;
    hops[v] = v == source ? 0 : -1;
    stamp[v] = 0;
    bucket_stamp[v] = 0;
  }
  if (first_thread() == 0) {
    near_v[0] = source;
    near_d[0] = 0;
    c->lowered = c->near = c->far = c->inspected = c->reached = c->max_hops = 0;
    c->invalid = c->far_min = ~0ull;
  }
}

// segments per frontier vertex; the frontier's degree sum is the pass's inspected entries
__global__ void segments_kernel(uint64_t nf, const uint32_t *queue, WAdj adj, uint64_t *seg_count, Counters *c) {
  unsigned long long deg_sum = 0;
  for (uint64_t i = first_thread(); i < ((nf + 31) & ~31ull); i += thread_count()) {
    uint64_t d = 0;
    if (i < nf) {
      d = adj.degree(queue[i]);
      seg_count[i] = (d + kSegEdges - 1) / kSegEdges;
    }
    deg_sum += d;
  }
  for (int o = 16; o > 0; o >>= 1) deg_sum += __shfl_xor_sync(kFull, deg_sum, o);
  if ((threadIdx.x & 31) == 0 && deg_sum) atomicAdd(&c->inspected, deg_sum);
}

// One warp per (frontier vertex, segment).  kTight = false: relax every valid entry with the vertex's frozen distance,
// list each lowered vertex once per pass.  kTight = true: the hop BFS over tight entries (final distances).
template <bool kTight>
__global__ void __launch_bounds__(kThreads) relax_kernel(uint64_t nf, const uint32_t *queue, const uint64_t *frozen,
                                                         const uint64_t *seg_scan, WAdj adj, uint64_t *dist,
                                                         uint32_t *stamp, uint32_t pass, int32_t *hops,
                                                         uint32_t *lowered, Counters *c) {
  const int lane = threadIdx.x & 31;
  const uint64_t warps_total = static_cast<uint64_t>(gridDim.x) * (kThreads / 32);
  const uint64_t total_items = seg_scan[nf];
  unsigned long long invalid = ~0ull;
  for (uint64_t item = static_cast<uint64_t>(blockIdx.x) * (kThreads / 32) + (threadIdx.x >> 5); item < total_items;
       item += warps_total) {
    uint64_t lo = 0, hi = nf;  // largest i with seg_scan[i] <= item
    while (lo + 1 < hi) {
      const uint64_t mid = (lo + hi) >> 1;
      if (seg_scan[mid] <= item) lo = mid; else hi = mid;
    }
    const uint32_t u = queue[lo];
    const uint64_t du = kTight ? dist[u] : frozen[lo];
    const uint64_t deg = adj.degree(u);
    const uint64_t k0 = (item - seg_scan[lo]) * kSegEdges;
    const uint64_t k1 = (k0 + kSegEdges < deg) ? k0 + kSegEdges : deg;
    for (uint64_t kb = k0; kb < k1; kb += 32) {
      const uint64_t k = kb + lane;
      bool take = false;
      uint32_t v = 0;
      if (k < k1) {
        uint64_t w = 0;
        adj.entry(u, k, &v, &w);
        if (w > kInfBits) {
          invalid = min(invalid, static_cast<unsigned long long>(w & kIndexMask));
        } else {
          const uint64_t nd = add_bits(du, w);
          if (kTight) {
            take = nd == dist[v] && hops[v] == -1 && atomicCAS(hops + v, -1, static_cast<int32_t>(pass)) == -1;
          } else if (nd < dist[v]) {
            const unsigned long long old = atomicMin(reinterpret_cast<unsigned long long *>(dist + v), nd);
            take = nd < old && atomicExch(stamp + v, pass) != pass;
          }
        }
      }
      warp_push(take, v, lowered, &c->lowered);
    }
  }
  if (!kTight) {
    for (int o = 16; o > 0; o >>= 1) invalid = min(invalid, __shfl_xor_sync(kFull, invalid, o));
    if (lane == 0 && invalid != ~0ull) atomicMin(&c->invalid, invalid);
  }
}

// The lowered vertices' final values: below T -> near pile (with the value frozen for the next pass), else the far pile
// once per bucket.  Bounded runs (T = kUnreached) send everything to the near pile and record hops = pass.
__global__ void classify_kernel(const uint32_t *lowered, const uint64_t *dist, uint64_t T, uint32_t bucket,
                                int bounded, uint32_t pass, int32_t *hops, uint32_t *bucket_stamp, uint32_t *near_v,
                                uint64_t *near_d, uint32_t *far, Counters *c) {
  const uint64_t count = c->lowered;
  for (uint64_t i = first_thread(); i < count; i += thread_count()) {
    const uint32_t v = lowered[i];
    const uint64_t d = dist[v];
    if (bounded) hops[v] = static_cast<int32_t>(pass);
    if (d < T) {
      const unsigned long long at = atomicAdd(&c->near, 1ull);
      near_v[at] = v;
      near_d[at] = d;
    } else if (atomicExch(bucket_stamp + v, bucket) != bucket) {
      far[atomicAdd(&c->far, 1ull)] = v;
    }
  }
}

__global__ void far_min_kernel(uint64_t nfar, const uint32_t *far, const uint64_t *dist, uint64_t T, Counters *c) {
  unsigned long long best = ~0ull;
  for (uint64_t i = first_thread(); i < ((nfar + 31) & ~31ull); i += thread_count()) {
    if (i < nfar) {
      const uint64_t d = dist[far[i]];
      if (d >= T) best = min(best, static_cast<unsigned long long>(d));
    }
  }
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(kFull, best, o));
  if ((threadIdx.x & 31) == 0 && best != ~0ull) atomicMin(&c->far_min, best);
}

// Far entries below the finished bucket's T were handled through the near pile; [T, T_next) -> near; the rest stays.
__global__ void split_kernel(uint64_t nfar, const uint32_t *far, const uint64_t *dist, uint64_t T, uint64_t T_next,
                             uint32_t bucket_next, uint32_t *bucket_stamp, uint32_t *near_v, uint64_t *near_d,
                             uint32_t *far_next, Counters *c) {
  for (uint64_t i = first_thread(); i < nfar; i += thread_count()) {
    const uint32_t v = far[i];
    const uint64_t d = dist[v];
    if (d < T) continue;
    if (d < T_next) {
      const unsigned long long at = atomicAdd(&c->near, 1ull);
      near_v[at] = v;
      near_d[at] = d;
    } else {
      bucket_stamp[v] = bucket_next;
      far_next[atomicAdd(&c->far, 1ull)] = v;
    }
  }
}

__global__ void output_kernel(uint64_t n, uint32_t source, const uint64_t *dist, const int32_t *hops, double *dist_out,
                              int32_t *hops_out, Counters *c) {
  unsigned long long reached = 0, max_hops = 0;
  for (uint64_t v = first_thread(); v < ((n + 31) & ~31ull); v += thread_count()) {
    if (v >= n) continue;
    const bool yielded = v != source && dist[v] != kUnreached;
    dist_out[v] = yielded ? __longlong_as_double(static_cast<long long>(dist[v])) : __longlong_as_double(0x7FF8000000000000ll);
    hops_out[v] = yielded ? hops[v] : -1;
    if (yielded) {
      ++reached;
      max_hops = max(max_hops, static_cast<unsigned long long>(hops[v]));
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    reached += __shfl_xor_sync(kFull, reached, o);
    max_hops = max(max_hops, __shfl_xor_sync(kFull, max_hops, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (reached) atomicAdd(&c->reached, reached);
    if (max_hops) atomicMax(&c->max_hops, max_hops);
  }
}

uint64_t bits_of(double x) {
  uint64_t b;
  std::memcpy(&b, &x, sizeof b);
  return b;
}
double double_of(uint64_t b) {
  double x;
  std::memcpy(&x, &b, sizeof x);
  return x;
}

// The end of the delta-wide bucket holding x (strictly above x); kUnreached once it would reach +inf.
uint64_t bucket_end(uint64_t x_bits, double delta) {
  if (x_bits >= kInfBits) return kUnreached;
  const double x = double_of(x_bits);
  double t = (std::floor(x / delta) + 1.0) * delta;
  if (!(t > x)) t = std::nextafter(x, HUGE_VAL);
  return std::isinf(t) ? kUnreached : bits_of(t);
}

// 1 in *bad unless sorted key e is (row, adj[e]) with e inside row's list: the sorted COO is the graph's list.
__global__ void same_pairs_kernel(uint64_t m, uint64_t n, const uint64_t *key, const uint64_t *ptr,
                                  const uint32_t *adj, int *bad) {
  for (uint64_t e = first_thread(); e < m; e += thread_count()) {
    const uint64_t row = key[e] >> 32;
    if (row >= n || e < ptr[row] || e >= ptr[row + 1] || adj[e] != static_cast<uint32_t>(key[e])) *bad = 1;
  }
}

// One side: the host's (row << 32 | neighbour) keys sorted with the weight bits as values, straight into *out, so
// *out lines up with the side's sorted list.  Staging: two key buffers and one value buffer (24 B per edge) plus
// cub's temporary, freed before the call returns.
int sort_side(mgb200_bfs_graph &g, const std::vector<uint64_t> &host_key, const std::vector<uint64_t> &w,
              const uint64_t *ptr, const uint32_t *adj, double *out) {
  const uint64_t m = g.m;
  cudaStream_t st = g.stream;
  DeviceBuffers tmp;
  uint64_t *key = nullptr, *key_alt = nullptr, *val_alt = nullptr;
  int *bad = nullptr;
  uint64_t *val = reinterpret_cast<uint64_t *>(out);
  MGB_CUDA(tmp.alloc(&key, m));
  MGB_CUDA(tmp.alloc(&key_alt, m));
  MGB_CUDA(tmp.alloc(&val_alt, m));
  MGB_CUDA(tmp.alloc(&bad, 1));
  MGB_CUDA(cudaMemcpyAsync(key, host_key.data(), m * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  MGB_CUDA(cudaMemcpyAsync(val, w.data(), m * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  MGB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), st));
  cub::DoubleBuffer<uint64_t> kb(key, key_alt), vb(val, val_alt);
  int bits = 1;
  while (bits < 32 && (g.n >> bits) != 0) ++bits;
  size_t bytes = 0;
  MGB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, kb, vb, m, 0, 32 + bits, st));
  char *t = nullptr;
  MGB_CUDA(tmp.alloc(&t, bytes));
  MGB_CUDA(cub::DeviceRadixSort::SortPairs(t, bytes, kb, vb, m, 0, 32 + bits, st));
  if (vb.Current() != val)
    MGB_CUDA(cudaMemcpyAsync(val, vb.Current(), m * sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
  same_pairs_kernel<<<blocks_for(m, g.sm_count, 16), kThreads, 0, st>>>(m, g.n, kb.Current(), ptr, adj, bad);
  MGB_CUDA(cudaGetLastError());
  int bad_host = 0;
  MGB_CUDA(cudaMemcpyAsync(&bad_host, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  if (bad_host) {
    set_error("wsp: set_weights needs the COO the graph was built from (its (from, to) pairs differ from the graph's)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  return MGB200_OK;
}

}  // namespace
}  // namespace mgb200

using namespace mgb200;

extern "C" {

int mgb200_bfs_graph_set_weights(mgb200_bfs_graph *g, uint64_t m, const uint64_t *from, const uint64_t *to,
                                 const double *weight) {
  if (!g || m != g->m || (m > 0 && (!from || !to || !weight))) {
    set_error("wsp: set_weights needs the graph's own COO (m equal to its edge count, non-null arrays)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  if (m > kIndexMask) {
    set_error("wsp: more than 2^51 edges");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  for (uint64_t e = 0; e < m; ++e) {
    if (from[e] >= g->n || to[e] >= g->n) {
      set_error("edge endpoint out of range (>= number_of_nodes)");
      return MGB200_ERR_INVALID_ARGUMENT;
    }
  }
  MGB_CUDA(cudaSetDevice(g->device));
  // the old weights go first: a failure below leaves the graph without weights, never with a mix of two sets
  auto clear = [g]() {
    cudaFree(g->out_w);
    cudaFree(g->in_w);
    g->out_w = g->in_w = nullptr;
    g->mean_weight = 0.0;
  };
  clear();
  if (m == 0) return MGB200_OK;
  std::vector<uint64_t> w(m), key(m);
  double sum = 0.0;
  uint64_t finite = 0;
  for (uint64_t e = 0; e < m; ++e) {
    const double x = weight[e];
    if (std::isnan(x) || x < 0.0) {
      w[e] = kInvalidTag | e;
    } else {
      w[e] = x == 0.0 ? 0ull : bits_of(x);  // -0.0 -> +0.0
      if (std::isfinite(x)) {
        sum += x;
        ++finite;
      }
    }
  }
  auto body = [&]() -> int {
    MGB_CUDA(cudaMalloc(&g->out_w, m * sizeof(double)));
    for (uint64_t e = 0; e < m; ++e) key[e] = (from[e] << 32) | to[e];
    int rc = sort_side(*g, key, w, g->out_ptr, g->out_adj, g->out_w);
    if (rc) return rc;
    MGB_CUDA(cudaMalloc(&g->in_w, m * sizeof(double)));
    for (uint64_t e = 0; e < m; ++e) key[e] = (to[e] << 32) | from[e];
    return sort_side(*g, key, w, g->in_ptr, g->in_adj, g->in_w);
  };
  const int rc = body();
  if (rc) {
    clear();
    return rc;
  }
  g->mean_weight = finite ? sum / static_cast<double>(finite) : 0.0;
  return MGB200_OK;
}

int mgb200_wsp_run(mgb200_bfs_graph *g, uint64_t source, int direction, int64_t upper_bound,
                   int (*should_abort)(void *user), void *abort_user, double *dist_out, int32_t *hops_out,
                   mgb200_wsp_stats *stats_out) {
  if (!g || (g->n > 0 && (!dist_out || !hops_out)) || direction < MGB200_BFS_OUT || direction > MGB200_BFS_BOTH) {
    set_error("wsp: invalid argument");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  if (upper_bound < 1) {
    set_error("Maximum depth in weighted shortest path expansion must be at least 1.");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  if (source >= g->n) {
    set_error("wsp: source vertex out of range");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  if (g->m > 0 && (!g->out_w || !g->in_w)) {
    set_error("wsp: the graph has no weights (call mgb200_bfs_graph_set_weights first)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  MGB_CUDA(cudaSetDevice(g->device));
  cudaStream_t st = g->stream;
  const uint64_t n = g->n;
  const bool bounded = upper_bound != MGB200_WSP_UNBOUNDED;
  mgb200_wsp_stats stats{};
  stats.invalid_edge = UINT64_MAX;
  const auto *ow = reinterpret_cast<const uint64_t *>(g->out_w), *iw = reinterpret_cast<const uint64_t *>(g->in_w);
  WAdj adj{};
  if (direction == MGB200_BFS_OUT) adj = WAdj{g->out_ptr, g->out_adj, ow, nullptr, nullptr, nullptr};
  else if (direction == MGB200_BFS_IN) adj = WAdj{g->in_ptr, g->in_adj, iw, nullptr, nullptr, nullptr};
  else adj = WAdj{g->out_ptr, g->out_adj, ow, g->in_ptr, g->in_adj, iw};

  // bucket width (Davidson et al.): warp width times the mean weight over the mean walked degree
  const double mean_degree = static_cast<double>(direction == MGB200_BFS_BOTH ? 2 * g->m : g->m) /
                             static_cast<double>(std::max<uint64_t>(n, 1));
  double delta = 32.0 * g->mean_weight / std::max(1.0, mean_degree);
  if (!(delta > 0.0) || !std::isfinite(delta)) delta = 1.0;
  // MGB200_WSP_DELTA: a finite width > 0 replaces the heuristic (anything else is ignored).  The width changes the
  // work only, never a result, so tests use it to put distances on bucket ends and to force many or one bucket.
  if (const char *s = std::getenv("MGB200_WSP_DELTA")) {
    char *end = nullptr;
    const double v = std::strtod(s, &end);
    if (end != s && *end == '\0' && v > 0.0 && std::isfinite(v)) delta = v;
  }

  DeviceBuffers buf;
  uint64_t *dist = nullptr, *near_d[2] = {nullptr, nullptr};
  int32_t *hops = nullptr, *hops_dev_out = nullptr;
  uint32_t *stamp = nullptr, *bucket_stamp = nullptr, *lowered = nullptr, *near_v[2] = {nullptr, nullptr},
           *far[2] = {nullptr, nullptr};
  double *dist_dev_out = nullptr;
  Counters *counters = nullptr;
  MGB_CUDA(buf.alloc(&dist, n));
  MGB_CUDA(buf.alloc(&hops, n));
  MGB_CUDA(buf.alloc(&stamp, n));
  MGB_CUDA(buf.alloc(&bucket_stamp, n));
  MGB_CUDA(buf.alloc(&lowered, n));
  for (int i = 0; i < 2; ++i) {
    MGB_CUDA(buf.alloc(&near_v[i], n));
    MGB_CUDA(buf.alloc(&near_d[i], n));
    MGB_CUDA(buf.alloc(&far[i], n));
  }
  MGB_CUDA(buf.alloc(&dist_dev_out, n));
  MGB_CUDA(buf.alloc(&hops_dev_out, n));
  MGB_CUDA(buf.alloc(&counters, 1));
  Counters host{};

  auto sync_counters = [&]() -> int {
    MGB_CUDA(cudaGetLastError());
    MGB_CUDA(cudaMemcpyAsync(&host, counters, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    MGB_CUDA(cudaStreamSynchronize(st));
    return MGB200_OK;
  };
  auto aborted = [&]() { return should_abort && should_abort(abort_user) != 0; };
  // segments + scan + relax over `nf` frontier vertices
  auto relax = [&](bool tight, uint64_t nf, const uint32_t *queue, const uint64_t *frozen, uint32_t pass) -> int {
    segments_kernel<<<blocks_for(nf, g->sm_count, 16), kThreads, 0, st>>>(nf, queue, adj, g->seg_count, counters);
    MGB_CUDA(cub::DeviceScan::ExclusiveSum(g->cub_tmp, g->cub_tmp_bytes, g->seg_count, g->seg_scan, nf + 1, st));
    if (tight)
      relax_kernel<true><<<g->sm_count * 8, kThreads, 0, st>>>(nf, queue, frozen, g->seg_scan, adj, dist, stamp, pass,
                                                              hops, lowered, counters);
    else
      relax_kernel<false><<<g->sm_count * 8, kThreads, 0, st>>>(nf, queue, frozen, g->seg_scan, adj, dist, stamp, pass,
                                                               hops, lowered, counters);
    stats.kernel_launches += 3;
    return MGB200_OK;
  };

  MGB_CUDA(cudaEventRecord(g->ev0, st));
  init_kernel<<<blocks_for(n, g->sm_count, 16), kThreads, 0, st>>>(n, static_cast<uint32_t>(source), dist, hops, stamp,
                                                               bucket_stamp, near_v[0], near_d[0], counters);
  stats.kernel_launches++;
  uint64_t nn = 1, nfar = 0;
  int cur = 0, fc = 0;
  uint32_t pass = 0, bucket = 1;
  uint64_t T = bounded ? kUnreached : bucket_end(0, delta);
  for (;;) {
    while (nn > 0 && !(bounded && static_cast<int64_t>(pass) >= upper_bound)) {
      if (aborted()) return set_error("procedure aborted by the host"), MGB200_ERR_ABORTED;
      ++pass;
      MGB_CUDA(cudaMemsetAsync(&counters->lowered, 0, 2 * sizeof(unsigned long long), st));  // lowered, near
      int rc = relax(false, nn, near_v[cur], near_d[cur], pass);
      if (rc) return rc;
      classify_kernel<<<blocks_for(nn * 4, g->sm_count, 16), kThreads, 0, st>>>(
          lowered, dist, T, bucket, bounded ? 1 : 0, pass, hops, bucket_stamp, near_v[cur ^ 1], near_d[cur ^ 1],
          far[fc], counters);
      stats.kernel_launches++;
      rc = sync_counters();
      if (rc) return rc;
      stats.relaxations += host.lowered;
      nn = host.near;
      nfar = host.far;
      cur ^= 1;
    }
    if (bounded || nfar == 0) break;
    if (aborted()) return set_error("procedure aborted by the host"), MGB200_ERR_ABORTED;
    MGB_CUDA(cudaMemsetAsync(&counters->far_min, 0xff, sizeof(unsigned long long), st));
    far_min_kernel<<<blocks_for(nfar, g->sm_count, 16), kThreads, 0, st>>>(nfar, far[fc], dist, T, counters);
    stats.kernel_launches++;
    int rc = sync_counters();
    if (rc) return rc;
    if (host.far_min == ~0ull) break;  // every far entry was handled through the near pile
    const uint64_t T_next = bucket_end(host.far_min, delta);
    MGB_CUDA(cudaMemsetAsync(&counters->near, 0, 2 * sizeof(unsigned long long), st));  // near, far
    split_kernel<<<blocks_for(nfar, g->sm_count, 16), kThreads, 0, st>>>(nfar, far[fc], dist, T, T_next, bucket + 1,
                                                                     bucket_stamp, near_v[cur], near_d[cur],
                                                                     far[fc ^ 1], counters);
    stats.kernel_launches++;
    rc = sync_counters();
    if (rc) return rc;
    nn = host.near;
    nfar = host.far;
    fc ^= 1;
    T = T_next;
    ++bucket;
    ++stats.buckets;
  }
  stats.rounds = pass;
  if (!bounded) {
    stats.buckets++;  // the first bucket
    // hops: level-synchronous BFS from the source over the tight entries
    uint32_t *queue[2] = {near_v[0], near_v[1]};
    const uint32_t s32 = static_cast<uint32_t>(source);
    MGB_CUDA(cudaMemcpyAsync(queue[0], &s32, sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    uint64_t nq = 1;
    int q = 0;
    for (uint32_t level = 1; nq > 0; ++level) {
      if (aborted()) return set_error("procedure aborted by the host"), MGB200_ERR_ABORTED;
      MGB_CUDA(cudaMemsetAsync(&counters->lowered, 0, sizeof(unsigned long long), st));
      int rc = relax(true, nq, queue[q], nullptr, level);
      if (rc) return rc;
      rc = sync_counters();
      if (rc) return rc;
      nq = host.lowered;
      // the BFS writes its next level into the lowered list; copy it into the other queue
      if (nq) MGB_CUDA(cudaMemcpyAsync(queue[q ^ 1], lowered, nq * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
      q ^= 1;
    }
  }
  output_kernel<<<blocks_for(n, g->sm_count, 16), kThreads, 0, st>>>(n, static_cast<uint32_t>(source), dist, hops,
                                                                 dist_dev_out, hops_dev_out, counters);
  stats.kernel_launches++;
  MGB_CUDA(cudaEventRecord(g->ev1, st));
  MGB_CUDA(cudaMemcpyAsync(dist_out, dist_dev_out, n * sizeof(double), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaMemcpyAsync(hops_out, hops_dev_out, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  int rc = sync_counters();
  if (rc) return rc;
  float ms = 0.f;
  MGB_CUDA(cudaEventElapsedTime(&ms, g->ev0, g->ev1));
  stats.run_ms = ms;
  stats.delta = bounded ? 0.0 : delta;
  stats.reached = host.reached;
  stats.hop_levels = static_cast<uint32_t>(host.max_hops);
  stats.entries_inspected = host.inspected;
  stats.invalid_edge = host.invalid;
  if (stats_out) *stats_out = stats;
  if (host.invalid != ~0ull) {
    set_error("wsp: an evaluated edge weight is negative or not a number (COO index " + std::to_string(host.invalid) +
              ")");
    return MGB200_ERR_INVALID_WEIGHT;
  }
  return MGB200_OK;
}

int mgb200_weighted_shortest_paths(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                   const double *weight, uint64_t source, int direction, int64_t upper_bound,
                                   double *dist_out, int32_t *hops_out) {
  mgb200_bfs_graph *g = nullptr;
  int rc = mgb200_bfs_graph_create_host(0, n, m, from, to, &g);
  if (rc) return rc;
  rc = mgb200_bfs_graph_set_weights(g, m, from, to, weight);
  if (!rc) rc = mgb200_wsp_run(g, source, direction, upper_bound, nullptr, nullptr, dist_out, hops_out, nullptr);
  mgb200_bfs_graph_destroy(g);
  return rc;
}

}  // extern "C"

// memgraph_b200/csrc/biconnectivity.cu -- bridges and biconnected components for sm_90a (include/mgb200_bfs.h).
//
// Semantics: the partition of the reference's bridges.get and biconnected_components.get (mage/cpp/bridges_module,
// mage/cpp/biconnected_components_module; restated in oracle/biconnectivity_oracle.c), which run a recursive
// Hopcroft-Tarjan DFS on one host thread.  Here both come from one spanning forest (Tarjan-Vishkin), integer work only:
//   roots     the union-find of wcc.cu over the COO: every component's root is its smallest id
//   forest    undirected_walk.cuh's level-synchronous BFS over the undirected view (out-list, then in-list) from all
//             roots at once; the parent of a vertex is its smallest-id neighbour in the previous level
//   size      levels bottom-up, atomicAdd of each subtree size into the parent
//   pre       the non-roots sorted by (parent, id) once (stable cub radix sort on the parent); a vertex's sibling offset
//             is the exclusive sum of its earlier siblings' sizes; levels top-down, pre(v) = pre(parent) + 1 + offset.
//             Roots take their components' offsets in root order
//   low/high  local(v) = min / max of pre(w) over v's undirected entries and pre(v), with exactly one occurrence of
//             parent(v) left out (further copies count: a doubled tree edge is a cycle); levels bottom-up with
//             atomicMin / atomicMax into the parent
//   bridge    tree edge (parent(v), v) is a bridge iff low(v) >= pre(v) and high(v) < pre(v) + size(v)
//   blocks    union-find over the tree edges, named by their child: link e(u), e(w) for every non-loop edge whose ends
//             are unrelated (neither an ancestor of the other); link e(v), e(p) for every tree edge (p, v), p not a
//             root, with low(v) < pre(p) or high(v) >= pre(p) + size(p)
//   per edge  x = the endpoint with the larger pre; bridge = bridge(x) && parent(x) is the other end; block = e(x).
//             Blocks are numbered in the order of their first edge in the COO (an exclusive scan of first-edge flags)
// The entry scans are undirected_walk.cuh's: a thread per vertex up to kThreadEntries entries, a warp up to
// kWarpEntries and a block above.
// The forest costs one host round trip per BFS level, and every sweep one launch per level: deep forests (long paths)
// are launch-bound, see DESIGN.md section 9.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "bfs_graph.hpp"
#include "core.hpp"
#include "mgb200_bfs.h"
#include "undirected_walk.cuh"
#include "union_find.cuh"

namespace mgb200 {
namespace {

struct Counters {
  Split split[2];  // BFS level L uses split[L & 1]; its thread kernel clears the other for level L + 1
  unsigned long long inspected;
  unsigned long long bridges;
  unsigned long long components;
  unsigned long long trees;
};

__device__ __forceinline__ bool is_ancestor(uint32_t a, uint32_t b, const uint32_t *pre, const uint32_t *size) {
  return pre[a] <= pre[b] && pre[b] < pre[a] + size[a];
}

// ---- entry scans: an op walks the entries [rank, degree) of u with stride `width` ---------------------------------

struct LocalOp {  // min / max of pre over the entries, one occurrence of the tree parent left out
  Lists g;
  const uint32_t *pre;
  const uint32_t *tree_parent;
  uint32_t *low;
  uint32_t *high;
  __device__ __forceinline__ static uint64_t copies(const uint32_t *adj, uint64_t begin, uint64_t end, uint32_t x) {
    uint64_t lo = begin, hi = end;  // lower bound of x in the sorted row
    while (lo < hi) {
      const uint64_t mid = (lo + hi) >> 1;
      if (adj[mid] < x) lo = mid + 1; else hi = mid;
    }
    uint64_t k = lo;
    while (k < end && k - lo < 2 && adj[k] == x) ++k;  // two copies are enough to know
    return k - lo;
  }
  __device__ __forceinline__ void operator()(uint32_t u, uint64_t rank, uint64_t width) const {
    const uint32_t p = tree_parent[u];
    const uint64_t ob = g.out_ptr[u], od = g.out_ptr[u + 1] - ob;
    const uint64_t ib = g.in_ptr[u], id = g.in_ptr[u + 1] - ib;
    uint32_t mn = kNone, mx = 0;
    for (uint64_t i = rank; i < od + id; i += width) {
      const uint32_t w = i < od ? g.out_adj[ob + i] : g.in_adj[ib + (i - od)];
      if (w == p) continue;
      const uint32_t pw = pre[w];
      mn = min(mn, pw);
      mx = max(mx, pw);
    }
    if (rank == 0 && p != kNone &&
        copies(g.out_adj, ob, ob + od, p) + copies(g.in_adj, ib, ib + id, p) >= 2) {  // a parallel tree edge
      mn = min(mn, pre[p]);
      mx = max(mx, pre[p]);
    }
    if (mn != kNone) atomicMin(low + u, mn);
    if (mx != 0) atomicMax(high + u, mx);
  }
};

// ---- per-vertex and per-edge passes ---------------------------------------------------------------------------------

__global__ void __launch_bounds__(kThreads) link_edges_kernel(uint64_t m, const uint32_t *from, const uint32_t *to,
                                                              uint32_t *parent) {
  for (uint64_t e = first_thread(); e < m; e += thread_count())
    if (from[e] != to[e]) link(from[e], to[e], parent);
}

__global__ void __launch_bounds__(kThreads) size_level_kernel(uint64_t lo, uint64_t hi, const uint32_t *order,
                                                              const uint32_t *tree_parent, uint32_t *size) {
  for (uint64_t i = lo + first_thread(); i < hi; i += thread_count()) {
    const uint32_t v = order[i];
    atomicAdd(size + tree_parent[v], size[v]);
  }
}

struct RootSize {  // the size of a root's tree, 0 for other vertices
  const uint32_t *tree_parent;
  const uint32_t *size;
  __device__ __forceinline__ uint32_t operator()(uint64_t v) const { return tree_parent[v] == kNone ? size[v] : 0u; }
};

struct SortedSize {  // the size of the i-th vertex in (parent, id) order
  const uint32_t *sorted;
  const uint32_t *size;
  __device__ __forceinline__ uint32_t operator()(uint64_t i) const { return size[sorted[i]]; }
};

// Roots: pre = the exclusive sum of the tree sizes before them; counts the trees with an edge.
__global__ void __launch_bounds__(kThreads) root_pre_kernel(uint64_t n, const uint32_t *tree_parent,
                                                            const uint32_t *size, const uint32_t *scan, uint32_t *pre,
                                                            Counters *counters) {
  unsigned long long trees = 0;
  for (uint64_t v = first_thread(); v < warp_rounded(n); v += thread_count()) {
    if (v >= n || tree_parent[v] != kNone) continue;
    pre[v] = scan[v];
    trees += size[v] > 1;
  }
  add_warp_sum(trees, &counters->trees);
}

// run_start[p] = the position of p's first child in (parent, id) order.
__global__ void __launch_bounds__(kThreads) run_start_kernel(uint64_t n, const uint32_t *keys, uint32_t *run_start) {
  for (uint64_t i = first_thread(); i < n; i += thread_count()) {
    const uint32_t p = keys[i];
    if (p != kNone && (i == 0 || keys[i - 1] != p)) run_start[p] = static_cast<uint32_t>(i);
  }
}

// Non-roots: pre = the sizes of the earlier siblings, completed by pre_level_kernel.
__global__ void __launch_bounds__(kThreads) sibling_kernel(uint64_t n, const uint32_t *keys, const uint32_t *sorted,
                                                           const uint32_t *run_start, const uint32_t *scan,
                                                           uint32_t *pre) {
  for (uint64_t i = first_thread(); i < n; i += thread_count()) {
    const uint32_t p = keys[i];
    if (p != kNone) pre[sorted[i]] = scan[i] - scan[run_start[p]];
  }
}

__global__ void __launch_bounds__(kThreads) pre_level_kernel(uint64_t lo, uint64_t hi, const uint32_t *order,
                                                             const uint32_t *tree_parent, uint32_t *pre) {
  for (uint64_t i = lo + first_thread(); i < hi; i += thread_count()) {
    const uint32_t v = order[i];
    pre[v] += pre[tree_parent[v]] + 1;
  }
}

__global__ void __launch_bounds__(kThreads) low_high_init_kernel(uint64_t n, const uint32_t *pre, uint32_t *low,
                                                                 uint32_t *high) {
  for (uint64_t v = first_thread(); v < n; v += thread_count()) low[v] = high[v] = pre[v];
}

__global__ void __launch_bounds__(kThreads) low_high_level_kernel(uint64_t lo, uint64_t hi, const uint32_t *order,
                                                                  const uint32_t *tree_parent, uint32_t *low,
                                                                  uint32_t *high) {
  for (uint64_t i = lo + first_thread(); i < hi; i += thread_count()) {
    const uint32_t v = order[i], p = tree_parent[v];
    atomicMin(low + p, low[v]);
    atomicMax(high + p, high[v]);
  }
}

// Blocks: non-loop edges between unrelated vertices, and tree edges whose child's subtree reaches past the parent's.
__global__ void __launch_bounds__(kThreads) link_unrelated_kernel(uint64_t m, const uint32_t *from, const uint32_t *to,
                                                                  const uint32_t *pre, const uint32_t *size,
                                                                  uint32_t *parent) {
  for (uint64_t e = first_thread(); e < m; e += thread_count()) {
    const uint32_t u = from[e], w = to[e];
    if (u != w && !is_ancestor(u, w, pre, size) && !is_ancestor(w, u, pre, size)) link(u, w, parent);
  }
}

__global__ void __launch_bounds__(kThreads) link_tree_kernel(uint64_t n, const uint32_t *tree_parent,
                                                             const uint32_t *pre, const uint32_t *size,
                                                             const uint32_t *low, const uint32_t *high,
                                                             uint32_t *parent) {
  for (uint64_t v = first_thread(); v < n; v += thread_count()) {
    const uint32_t p = tree_parent[v];
    if (p == kNone || tree_parent[p] == kNone) continue;
    if (low[v] < pre[p] || high[v] >= pre[p] + size[p]) link(static_cast<uint32_t>(v), p, parent);
  }
}

// Per edge: the bridge flag, the block (the union-find root of e(x)) and the block's first edge.
__global__ void __launch_bounds__(kThreads) classify_kernel(uint64_t m, const uint32_t *from, const uint32_t *to,
                                                            const uint32_t *tree_parent, const uint32_t *pre,
                                                            const uint32_t *size, const uint32_t *low,
                                                            const uint32_t *high, const uint32_t *parent,
                                                            uint8_t *bridge, uint32_t *block,
                                                            unsigned long long *first_edge, Counters *counters) {
  unsigned long long bridges = 0;
  for (uint64_t e = first_thread(); e < warp_rounded(m); e += thread_count()) {
    if (e >= m) continue;
    const uint32_t u = from[e], w = to[e];
    if (u == w) {
      bridge[e] = 0;
      block[e] = kNone;
      continue;
    }
    const uint32_t x = pre[u] > pre[w] ? u : w, other = x == u ? w : u;
    const bool is_bridge = tree_parent[x] == other && low[x] >= pre[x] && high[x] < pre[x] + size[x];
    bridge[e] = is_bridge ? 1 : 0;
    bridges += is_bridge;
    const uint32_t b = parent[x];
    block[e] = b;
    atomicMin(first_edge + b, static_cast<unsigned long long>(e));
  }
  add_warp_sum(bridges, &counters->bridges);
}

struct IsFirst {  // 32-bit flags: a block count fits, since blocks are named by vertices
  const uint32_t *block;
  const unsigned long long *first_edge;
  __device__ __forceinline__ uint32_t operator()(uint64_t e) const {
    return block[e] != kNone && first_edge[block[e]] == e ? 1u : 0u;
  }
};

// bcc holds the exclusive scan of the first-edge flags; every edge takes its block's first edge's value.  Only
// positions that are not a first edge are written, and only first-edge positions are read.
__global__ void __launch_bounds__(kThreads) number_kernel(uint64_t m, const uint32_t *block,
                                                          const unsigned long long *first_edge, int64_t *bcc,
                                                          Counters *counters) {
  unsigned long long firsts = 0;
  for (uint64_t e = first_thread(); e < warp_rounded(m); e += thread_count()) {
    if (e >= m) continue;
    const uint32_t b = block[e];
    if (b == kNone) {
      bcc[e] = -1;
      continue;
    }
    const unsigned long long f = first_edge[b];
    if (f == e) ++firsts; else bcc[e] = bcc[f];
  }
  add_warp_sum(firsts, &counters->components);
}

}  // namespace
}  // namespace mgb200

using namespace mgb200;

extern "C" {

int mgb200_biconnectivity_run(mgb200_bfs_graph *g, uint64_t m, const uint64_t *from, const uint64_t *to,
                              uint8_t *bridge_out, int64_t *bcc_out, mgb200_biconnectivity_stats *stats_out) {
  if (!g || m != g->m || (m > 0 && (!from || !to))) {
    set_error("biconnectivity: invalid argument (need a graph and its own COO: m equal to the graph's edge count)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  const uint64_t n = g->n;
  std::vector<uint32_t> f(m), t(m);
  for (uint64_t e = 0; e < m; ++e) {
    if (from[e] >= n || to[e] >= n) {
      set_error("biconnectivity: edge endpoint out of range (>= the graph's number of nodes)");
      return MGB200_ERR_INVALID_ARGUMENT;
    }
    f[e] = static_cast<uint32_t>(from[e]);
    t[e] = static_cast<uint32_t>(to[e]);
  }
  mgb200_biconnectivity_stats stats{};
  if (n == 0) {
    if (stats_out) *stats_out = stats;
    return MGB200_OK;
  }
  MGB_CUDA(cudaSetDevice(g->device));
  cudaStream_t st = g->stream;
  const Lists lists{g->out_ptr, g->out_adj, g->in_ptr, g->in_adj};
  uint32_t *order = g->queue[0], *work = g->queue[1];

  DeviceBuffers buf;
  uint32_t *d_from = nullptr, *d_to = nullptr, *uf = nullptr, *tree_parent = nullptr, *size = nullptr, *pre = nullptr,
           *low = nullptr, *high = nullptr, *keys = nullptr, *sorted = nullptr, *scan = nullptr, *block = nullptr;
  unsigned long long *first_edge = nullptr;
  uint8_t *bridge = nullptr;
  int64_t *bcc = nullptr;
  Counters *counters = nullptr;
  MGB_CUDA(buf.alloc(&d_from, m));
  MGB_CUDA(buf.alloc(&d_to, m));
  MGB_CUDA(buf.alloc(&uf, n));
  MGB_CUDA(buf.alloc(&tree_parent, n));
  MGB_CUDA(buf.alloc(&size, n));
  MGB_CUDA(buf.alloc(&pre, n));
  MGB_CUDA(buf.alloc(&low, n));
  MGB_CUDA(buf.alloc(&high, n));
  MGB_CUDA(buf.alloc(&keys, n));
  MGB_CUDA(buf.alloc(&sorted, n));
  MGB_CUDA(buf.alloc(&scan, n));
  MGB_CUDA(buf.alloc(&block, m));
  MGB_CUDA(buf.alloc(&first_edge, n));
  MGB_CUDA(buf.alloc(&bridge, m));
  MGB_CUDA(buf.alloc(&bcc, m));
  MGB_CUDA(buf.alloc(&counters, 1));
  uint32_t *iota = low, *run_start = high;  // both free until the low / high pass
  const auto root_sizes = thrust::make_transform_iterator(thrust::counting_iterator<uint64_t>(0),
                                                          RootSize{tree_parent, size});
  const auto sorted_sizes = thrust::make_transform_iterator(thrust::counting_iterator<uint64_t>(0),
                                                            SortedSize{sorted, size});
  const auto first_flags = thrust::make_transform_iterator(thrust::counting_iterator<uint64_t>(0),
                                                           IsFirst{block, first_edge});
  size_t root_bytes = 0, sort_bytes = 0, sibling_bytes = 0, number_bytes = 0;
  MGB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, root_bytes, root_sizes, scan, n, st));
  MGB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, tree_parent, keys, iota, sorted, n, 0, 32, st));
  MGB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, sibling_bytes, sorted_sizes, scan, n, st));
  if (m) MGB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, number_bytes, first_flags, bcc, m, st));
  const size_t tmp_bytes = std::max({root_bytes, sort_bytes, sibling_bytes, number_bytes});
  size_t bytes = tmp_bytes;
  void *cub_tmp = g->cub_tmp;  // the handle's scratch where it is large enough
  if (tmp_bytes > g->cub_tmp_bytes) {
    char *own = nullptr;
    MGB_CUDA(buf.alloc(&own, tmp_bytes));
    cub_tmp = own;
  }
  if (m) {
    MGB_CUDA(cudaMemcpyAsync(d_from, f.data(), m * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    MGB_CUDA(cudaMemcpyAsync(d_to, t.data(), m * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  }

  const int grid_n = blocks_for(n, g->sm_count, 8), grid_m = blocks_for(m, g->sm_count, 8);
  uint64_t launches = 0;
  MGB_CUDA(cudaEventRecord(g->ev0, st));
  MGB_CUDA(cudaMemsetAsync(counters, 0, sizeof(Counters), st));
  MGB_CUDA(cudaMemsetAsync(first_edge, 0xff, n * sizeof(unsigned long long), st));

  // roots: wcc.cu's union-find over the edges
  iota_kernel<<<grid_n, kThreads, 0, st>>>(n, uf);
  if (m) link_edges_kernel<<<grid_m, kThreads, 0, st>>>(m, d_from, d_to, uf);
  compress_kernel<<<grid_n, kThreads, 0, st>>>(n, uf);
  launches += m ? 3 : 2;

  // forest: one BFS level per round trip; level L's vertices are order[level[L], level[L + 1])
  std::vector<uint64_t> level;
  const int rc = bfs_forest(*g, uf, tree_parent, size, order, work, counters->split, &counters->inspected, &level,
                            &launches);
  if (rc) return rc;
  const uint32_t levels = static_cast<uint32_t>(level.size() - 2);  // the last entry closes an empty level
  if (level[levels] != n) {
    set_error("biconnectivity: the forest does not span the graph (internal error)");
    return MGB200_ERR_CUDA;
  }

  // subtree sizes, bottom-up
  for (uint32_t L = levels - 1; L >= 1; --L) {
    size_level_kernel<<<blocks_for(level[L + 1] - level[L], g->sm_count, 8), kThreads, 0, st>>>(
        level[L], level[L + 1], order, tree_parent, size);
    ++launches;
  }
  // preorder: roots in root order, siblings in id order, levels top-down
  MGB_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, bytes, root_sizes, scan, n, st));
  root_pre_kernel<<<grid_n, kThreads, 0, st>>>(n, tree_parent, size, scan, pre, counters);
  iota_kernel<<<grid_n, kThreads, 0, st>>>(n, iota);
  bytes = tmp_bytes;
  MGB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp, bytes, tree_parent, keys, iota, sorted, n, 0, 32, st));
  bytes = tmp_bytes;
  MGB_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, bytes, sorted_sizes, scan, n, st));
  run_start_kernel<<<grid_n, kThreads, 0, st>>>(n, keys, run_start);
  sibling_kernel<<<grid_n, kThreads, 0, st>>>(n, keys, sorted, run_start, scan, pre);
  launches += 4;
  for (uint32_t L = 1; L < levels; ++L) {
    pre_level_kernel<<<blocks_for(level[L + 1] - level[L], g->sm_count, 8), kThreads, 0, st>>>(
        level[L], level[L + 1], order, tree_parent, pre);
    ++launches;
  }
  // low / high: local values, then levels bottom-up
  low_high_init_kernel<<<grid_n, kThreads, 0, st>>>(n, pre, low, high);
  ++launches;
  MGB_CUDA(cudaMemsetAsync(&counters->split[0], 0, sizeof(Split), st));
  walk(*g, 0, n, nullptr, LocalOp{lists, pre, tree_parent, low, high}, work, &counters->split[0], nullptr,
       &counters->inspected, &launches);
  for (uint32_t L = levels - 1; L >= 1; --L) {
    low_high_level_kernel<<<blocks_for(level[L + 1] - level[L], g->sm_count, 8), kThreads, 0, st>>>(
        level[L], level[L + 1], order, tree_parent, low, high);
    ++launches;
  }
  // blocks: union-find over the tree edges, named by their child
  iota_kernel<<<grid_n, kThreads, 0, st>>>(n, uf);
  if (m) link_unrelated_kernel<<<grid_m, kThreads, 0, st>>>(m, d_from, d_to, pre, size, uf);
  link_tree_kernel<<<grid_n, kThreads, 0, st>>>(n, tree_parent, pre, size, low, high, uf);
  compress_kernel<<<grid_n, kThreads, 0, st>>>(n, uf);
  launches += m ? 4 : 3;
  if (m) {
    classify_kernel<<<grid_m, kThreads, 0, st>>>(m, d_from, d_to, tree_parent, pre, size, low, high, uf, bridge, block,
                                                 first_edge, counters);
    bytes = tmp_bytes;
    MGB_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, bytes, first_flags, bcc, m, st));
    number_kernel<<<grid_m, kThreads, 0, st>>>(m, block, first_edge, bcc, counters);
    launches += 2;
  }
  MGB_CUDA(cudaGetLastError());
  MGB_CUDA(cudaEventRecord(g->ev1, st));

  Counters host{};
  MGB_CUDA(cudaMemcpyAsync(&host, counters, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  if (bridge_out && m) MGB_CUDA(cudaMemcpyAsync(bridge_out, bridge, m, cudaMemcpyDeviceToHost, st));
  if (bcc_out && m) MGB_CUDA(cudaMemcpyAsync(bcc_out, bcc, m * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  float ms = 0.f;
  MGB_CUDA(cudaEventElapsedTime(&ms, g->ev0, g->ev1));
  stats.trees = host.trees;
  stats.forest_depth = levels - 1;
  stats.bridges = host.bridges;
  stats.components = host.components;
  stats.edges_inspected = host.inspected;
  stats.run_ms = ms;
  stats.kernel_launches = launches;
  if (stats_out) *stats_out = stats;
  return MGB200_OK;
}

int mgb200_bridges(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, uint8_t *bridge_out) {
  if (m > 0 && !bridge_out) {
    set_error("bridges: bridge_out is null");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  mgb200_bfs_graph *g = nullptr;
  int rc = mgb200_bfs_graph_create_host(0, n, m, from, to, &g);
  if (rc) return rc;
  rc = mgb200_biconnectivity_run(g, m, from, to, bridge_out, nullptr, nullptr);
  mgb200_bfs_graph_destroy(g);
  return rc;
}

int mgb200_biconnected_components(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, int64_t *bcc_out) {
  if (m > 0 && !bcc_out) {
    set_error("biconnected components: bcc_out is null");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  mgb200_bfs_graph *g = nullptr;
  int rc = mgb200_bfs_graph_create_host(0, n, m, from, to, &g);
  if (rc) return rc;
  rc = mgb200_biconnectivity_run(g, m, from, to, nullptr, bcc_out, nullptr);
  mgb200_bfs_graph_destroy(g);
  return rc;
}

}  // extern "C"

// memgraph_b200/csrc/wcc.cu -- weakly connected components for sm_90a (include/mgb200_bfs.h).
//
// Semantics: the reference's weakly_connected_components.get (mage/cpp/connectivity_module/connectivity_module.cpp:
// 41-84, restated in oracle/wcc_oracle.c): a BFS over the undirected view from every unvisited vertex in dense order,
// components numbered in that order.  A component's number is therefore the rank of its smallest dense id among the
// components' smallest ids.
//
// Afforest-style union-find on the out- and in-lists of the BFS device graph (one uint32 parent per vertex):
//   init      parent[v] = v
//   sample    kSampleRounds rounds; in round r every vertex links with entry r of its undirected list (the out-list,
//             then the in-list); each round is followed by a full compression
//   giant     the most frequent root among kSamples vertices chosen by a fixed hash is the giant component (ties: the
//             smaller root); its members are marked in a bit array
//   finish    every unmarked vertex links with the remaining entries of its undirected list, from position
//             kSampleRounds on.  An edge u -> w whose u is marked is still seen from w's in-list, so skipping the
//             giant's members loses no edge; then one more compression
//   label     flag = (parent[v] == v), exclusive scan of the flags, component[v] = scan[parent[v]] (number_sets,
//             union_find.cuh)
// The link hooks the larger of two roots under the smaller one with atomicCAS, and a compression only shortens paths,
// so parent[x] <= x always holds and every root is its component's smallest id, whatever order the threads link in.
// The output is integers: two runs are byte-identical.  The finish runs a thread per vertex up to kThreadEntries
// remaining entries, a warp per vertex up to kWarpEntries and a block per vertex above that (RMAT in-degrees reach
// about 10^6 at scale 26).
#include <cub/cub.cuh>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "bfs_graph.hpp"
#include "core.hpp"
#include "mgb200_bfs.h"
#include "union_find.cuh"

namespace mgb200 {
namespace {

constexpr uint32_t kSampleRounds = 2;
constexpr uint32_t kSamples = 1024;
constexpr uint64_t kSampleSeed = 0x5eed5eed5eedull;
constexpr uint64_t kThreadEntries = 16;    // remaining entries a single thread walks
constexpr uint64_t kWarpEntries = 4096;    // above this, a block (8 warps) per vertex

struct Lists {  // the undirected view: out-list, then in-list
  const uint64_t *out_ptr;
  const uint32_t *out_adj;
  const uint64_t *in_ptr;
  const uint32_t *in_adj;
};

struct Counters {
  unsigned long long inspected;
  unsigned long long skipped;
  unsigned int mid;    // vertices queued for a warp each (front of the work list)
  unsigned int heavy;  // vertices queued for a block each (back of the work list)
};

// Entry i of v's undirected list (i < out-degree + in-degree).
__device__ __forceinline__ uint32_t entry(const Lists &g, uint64_t out_begin, uint64_t out_deg, uint64_t in_begin,
                                          uint64_t i) {
  return i < out_deg ? g.out_adj[out_begin + i] : g.in_adj[in_begin + (i - out_deg)];
}

__global__ void __launch_bounds__(kThreads) init_kernel(uint64_t n, uint32_t *parent) {
  for (uint64_t v = first_thread(); v < n; v += thread_count()) parent[v] = static_cast<uint32_t>(v);
}

__global__ void __launch_bounds__(kThreads) sample_kernel(uint64_t n, Lists g, uint32_t round, uint32_t *parent,
                                                          Counters *counters) {
  unsigned long long inspected = 0;
  for (uint64_t v = first_thread(); v < warp_rounded(n); v += thread_count()) {
    if (v >= n) continue;
    const uint64_t ob = g.out_ptr[v], od = g.out_ptr[v + 1] - ob;
    const uint64_t ib = g.in_ptr[v], id = g.in_ptr[v + 1] - ib;
    if (round < od + id) {
      link(static_cast<uint32_t>(v), entry(g, ob, od, ib, round), parent);
      ++inspected;
    }
  }
  add_warp_sum(inspected, &counters->inspected);
}

__device__ __forceinline__ uint64_t mix64(uint64_t z) {  // splitmix64 finaliser
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__global__ void sample_roots_kernel(uint64_t n, const uint32_t *parent, uint32_t *roots) {
  for (uint32_t i = threadIdx.x + blockIdx.x * blockDim.x; i < kSamples; i += blockDim.x * gridDim.x)
    roots[i] = parent[mix64(kSampleSeed + 0x9E3779B97F4A7C15ull * (i + 1)) % n];
}

// skip bit of v = (v is in the giant component), one 32-bit word per warp; counts the skipped vertices.
__global__ void __launch_bounds__(kThreads) mark_kernel(uint64_t n, const uint32_t *parent, uint32_t giant,
                                                        uint32_t *skip, Counters *counters) {
  unsigned long long skipped = 0;
  for (uint64_t v = first_thread(); v < warp_rounded(n); v += thread_count()) {
    const bool in_giant = v < n && parent[v] == giant;
    const unsigned bits = __ballot_sync(kFull, in_giant);
    if ((threadIdx.x & 31) == 0) {
      skip[v >> 5] = bits;
      skipped += __popc(bits);
    }
  }
  if ((threadIdx.x & 31) == 0 && skipped) atomicAdd(&counters->skipped, skipped);
}

// Unmarked vertices: a thread walks up to kThreadEntries remaining entries itself and queues longer lists.
__global__ void __launch_bounds__(kThreads) finish_kernel(uint64_t n, Lists g, const uint32_t *skip, uint32_t *parent,
                                                          uint32_t *work, Counters *counters) {
  unsigned long long inspected = 0;
  for (uint64_t v = first_thread(); v < warp_rounded(n); v += thread_count()) {
    if (v >= n || ((skip[v >> 5] >> (v & 31)) & 1u)) continue;
    const uint64_t ob = g.out_ptr[v], od = g.out_ptr[v + 1] - ob;
    const uint64_t ib = g.in_ptr[v], id = g.in_ptr[v + 1] - ib;
    const uint64_t deg = od + id;
    if (deg <= kSampleRounds) continue;
    const uint64_t remaining = deg - kSampleRounds;
    if (remaining <= kThreadEntries) {
      for (uint64_t i = kSampleRounds; i < deg; ++i) link(static_cast<uint32_t>(v), entry(g, ob, od, ib, i), parent);
      inspected += remaining;
    } else if (remaining <= kWarpEntries) {
      work[atomicAdd(&counters->mid, 1u)] = static_cast<uint32_t>(v);
    } else {
      work[n - 1 - atomicAdd(&counters->heavy, 1u)] = static_cast<uint32_t>(v);
    }
  }
  add_warp_sum(inspected, &counters->inspected);
}

// The remaining entries of v, split over `width` threads starting at `rank`.
__device__ __forceinline__ void finish_vertex(const Lists &g, uint32_t v, uint32_t rank, uint32_t width,
                                              uint32_t *parent) {
  const uint64_t ob = g.out_ptr[v], od = g.out_ptr[v + 1] - ob;
  const uint64_t ib = g.in_ptr[v], id = g.in_ptr[v + 1] - ib;
  for (uint64_t i = kSampleRounds + rank; i < od + id; i += width) link(v, entry(g, ob, od, ib, i), parent);
}

__device__ __forceinline__ uint64_t remaining_entries(const Lists &g, uint32_t v) {
  return g.out_ptr[v + 1] - g.out_ptr[v] + g.in_ptr[v + 1] - g.in_ptr[v] - kSampleRounds;
}

__global__ void __launch_bounds__(kThreads) finish_warp_kernel(Lists g, const uint32_t *work, uint32_t *parent,
                                                               Counters *counters) {
  const uint32_t count = counters->mid;
  const uint32_t lane = threadIdx.x & 31;
  unsigned long long inspected = 0;
  for (uint64_t w = first_thread() >> 5; w < count; w += thread_count() >> 5) {
    const uint32_t v = work[w];
    finish_vertex(g, v, lane, 32, parent);
    if (lane == 0) inspected += remaining_entries(g, v);
  }
  if (lane == 0 && inspected) atomicAdd(&counters->inspected, inspected);
}

__global__ void __launch_bounds__(kThreads) finish_block_kernel(uint64_t n, Lists g, const uint32_t *work,
                                                                uint32_t *parent, Counters *counters) {
  const uint32_t count = counters->heavy;
  unsigned long long inspected = 0;
  for (uint32_t b = blockIdx.x; b < count; b += gridDim.x) {
    const uint32_t v = work[n - 1 - b];
    finish_vertex(g, v, threadIdx.x, blockDim.x, parent);
    if (threadIdx.x == 0) inspected += remaining_entries(g, v);
  }
  if (threadIdx.x == 0 && inspected) atomicAdd(&counters->inspected, inspected);
}

// size[root] += members; the members of `giant` are summed per block first (one address would serialise the atomics).
__global__ void __launch_bounds__(kThreads) size_kernel(uint64_t n, const uint32_t *parent, uint32_t giant,
                                                        uint32_t *size) {
  __shared__ unsigned int block_giant;
  if (threadIdx.x == 0) block_giant = 0;
  __syncthreads();
  unsigned int mine = 0;
  for (uint64_t v = first_thread(); v < warp_rounded(n); v += thread_count()) {
    const uint32_t r = v < n ? parent[v] : giant;
    if (r == giant && v < n) ++mine;
    const unsigned peers = __match_any_sync(kFull, r);  // the lanes with the same root add once
    if (r != giant && (threadIdx.x & 31) == static_cast<unsigned>(__ffs(peers) - 1)) atomicAdd(size + r, __popc(peers));
  }
  if (mine) atomicAdd(&block_giant, mine);
  __syncthreads();
  if (threadIdx.x == 0 && block_giant) atomicAdd(size + giant, block_giant);
}

// The most frequent value; ties go to the smaller one.
uint32_t most_frequent(std::vector<uint32_t> values) {
  std::sort(values.begin(), values.end());
  uint32_t best = values.empty() ? 0 : values[0];
  size_t best_count = 0;
  for (size_t i = 0; i < values.size();) {
    size_t j = i;
    while (j < values.size() && values[j] == values[i]) ++j;
    if (j - i > best_count) {
      best = values[i];
      best_count = j - i;
    }
    i = j;
  }
  return best;
}

}  // namespace
}  // namespace mgb200

using namespace mgb200;

extern "C" {

int mgb200_wcc_run(mgb200_bfs_graph *g, int64_t *component_out, mgb200_wcc_stats *stats_out) {
  if (!g || (g->n > 0 && !component_out)) {
    set_error("weakly connected components: invalid argument (need a graph and a non-null component_out)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  mgb200_wcc_stats stats{};
  const uint64_t n = g->n;
  if (n == 0) {
    if (stats_out) *stats_out = stats;
    return MGB200_OK;
  }
  MGB_CUDA(cudaSetDevice(g->device));
  cudaStream_t st = g->stream;
  const Lists lists{g->out_ptr, g->out_adj, g->in_ptr, g->in_adj};

  DeviceBuffers buf;
  uint32_t *parent = nullptr, *skip = nullptr, *work = nullptr, *size = nullptr, *scan = nullptr, *roots = nullptr,
           *largest = nullptr;
  int64_t *component = nullptr;
  Counters *counters = nullptr;
  MGB_CUDA(buf.alloc(&parent, n));
  MGB_CUDA(buf.alloc(&skip, (n + 31) / 32));
  MGB_CUDA(buf.alloc(&work, n));
  MGB_CUDA(buf.alloc(&size, n));
  MGB_CUDA(buf.alloc(&scan, n));
  MGB_CUDA(buf.alloc(&roots, kSamples));
  MGB_CUDA(buf.alloc(&largest, 1));
  MGB_CUDA(buf.alloc(&component, n));
  MGB_CUDA(buf.alloc(&counters, 1));
  size_t scan_bytes = 0, max_bytes = 0;
  MGB_CUDA(number_sets(n, parent, scan, component, nullptr, &scan_bytes, 1, st));
  MGB_CUDA(cub::DeviceReduce::Max(nullptr, max_bytes, size, largest, n, st));
  char *cub_tmp = nullptr;
  MGB_CUDA(buf.alloc(&cub_tmp, std::max(scan_bytes, max_bytes)));

  const int grid = blocks_for(n, g->sm_count, 8);
  MGB_CUDA(cudaEventRecord(g->ev0, st));
  MGB_CUDA(cudaMemsetAsync(counters, 0, sizeof(Counters), st));
  MGB_CUDA(cudaMemsetAsync(size, 0, n * sizeof(uint32_t), st));
  init_kernel<<<grid, kThreads, 0, st>>>(n, parent);
  stats.kernel_launches++;
  for (uint32_t r = 0; r < kSampleRounds; ++r) {
    sample_kernel<<<grid, kThreads, 0, st>>>(n, lists, r, parent, counters);
    compress_kernel<<<grid, kThreads, 0, st>>>(n, parent);
    stats.kernel_launches += 2;
  }
  sample_roots_kernel<<<kSamples / kThreads, kThreads, 0, st>>>(n, parent, roots);
  stats.kernel_launches++;
  std::vector<uint32_t> sampled(kSamples);
  MGB_CUDA(cudaMemcpyAsync(sampled.data(), roots, kSamples * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  MGB_CUDA(cudaGetLastError());
  const uint32_t giant = most_frequent(sampled);

  mark_kernel<<<grid, kThreads, 0, st>>>(n, parent, giant, skip, counters);
  finish_kernel<<<grid, kThreads, 0, st>>>(n, lists, skip, parent, work, counters);
  finish_warp_kernel<<<blocks_for(n * 32, g->sm_count, 16), kThreads, 0, st>>>(lists, work, parent, counters);
  finish_block_kernel<<<g->sm_count * 8, kThreads, 0, st>>>(n, lists, work, parent, counters);
  compress_kernel<<<grid, kThreads, 0, st>>>(n, parent);
  stats.kernel_launches += 5;
  // the giant component's root after the finish is the sampled root's root: compression pointed it there
  uint32_t giant_root = giant;
  MGB_CUDA(cudaMemcpyAsync(&giant_root, parent + giant, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  size_kernel<<<grid, kThreads, 0, st>>>(n, parent, giant_root, size);
  stats.kernel_launches++;
  MGB_CUDA(cub::DeviceReduce::Max(cub_tmp, max_bytes, size, largest, n, st));
  MGB_CUDA(number_sets(n, parent, scan, component, cub_tmp, &scan_bytes, grid, st));  // scan + label_kernel
  stats.kernel_launches++;
  MGB_CUDA(cudaGetLastError());
  MGB_CUDA(cudaEventRecord(g->ev1, st));

  Counters host_counters{};
  uint32_t tail[2] = {0, 0}, largest_host = 0;  // scan[n - 1], parent[n - 1]
  MGB_CUDA(cudaMemcpyAsync(&host_counters, counters, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaMemcpyAsync(&tail[0], scan + n - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaMemcpyAsync(&tail[1], parent + n - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaMemcpyAsync(&largest_host, largest, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaMemcpyAsync(component_out, component, n * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  float ms = 0.f;
  MGB_CUDA(cudaEventElapsedTime(&ms, g->ev0, g->ev1));
  stats.components = static_cast<uint64_t>(tail[0]) + (tail[1] == n - 1 ? 1 : 0);
  stats.largest_component = largest_host;
  stats.skipped_vertices = host_counters.skipped;
  stats.edges_inspected = host_counters.inspected;
  stats.run_ms = ms;
  if (stats_out) *stats_out = stats;
  return MGB200_OK;
}

int mgb200_weakly_connected_components(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                       int64_t *component_out) {
  if (n > 0 && !component_out) {
    set_error("weakly connected components: component_out is null");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  mgb200_bfs_graph *g = nullptr;
  int rc = mgb200_bfs_graph_create_host(0, n, m, from, to, &g);
  if (rc) return rc;
  rc = mgb200_wcc_run(g, component_out, nullptr);
  mgb200_bfs_graph_destroy(g);
  return rc;
}

}  // extern "C"

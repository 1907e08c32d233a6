// memgraph_b200/csrc/bfs_graph.hpp -- the device graph behind the opaque mgb200_bfs_graph handle (include/mgb200_bfs.h).
// Shared by the breadth-first expansion (bfs.cu), which builds it, betweenness centrality (betweenness.cu), weakly
// connected components (wcc.cu), bridges and biconnected components (biconnectivity.cu), weighted shortest paths
// (wsp.cu), bipartite matching (bipartite_matching.cu) and strongly connected components (scc.cu), which walk the same
// CSR + CSC; also the grid-stride and warp helpers of their kernels.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "mgb200_bfs.h"

struct mgb200_bfs_graph {
  int device = 0;
  int sm_count = 0;
  cudaStream_t stream = nullptr;
  uint64_t n = 0, m = 0;
  uint64_t *out_ptr = nullptr, *in_ptr = nullptr;   // [n + 1]
  uint32_t *out_adj = nullptr, *in_adj = nullptr;   // [m], sorted inside a row
  double *out_w = nullptr, *in_w = nullptr;         // [m] weights aligned with out_adj / in_adj; null until
                                                    // mgb200_bfs_graph_set_weights (wsp.cu)
  double mean_weight = 0.0;                         // mean of the finite valid weights (wsp.cu's bucket width)
  int32_t *depth = nullptr;                         // [n]
  uint32_t *queue[2] = {nullptr, nullptr};          // [n] frontier vertex lists
  uint32_t *bitmap[2] = {nullptr, nullptr};         // [ceil(n/32)]
  uint64_t *seg_count = nullptr, *seg_scan = nullptr;  // [n + 1]
  unsigned long long *counters = nullptr;           // device: [0] next size [1] frontier degree sum [2] inspected [3] items
  unsigned long long *host_counters = nullptr;      // pinned
  void *cub_tmp = nullptr;
  size_t cub_tmp_bytes = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

namespace mgb200 {
namespace {

constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ uint64_t first_thread() { return static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; }
__device__ __forceinline__ uint64_t thread_count() { return static_cast<uint64_t>(gridDim.x) * blockDim.x; }

// Grid-stride loops that shuffle run whole warps (the bound is rounded up to a multiple of 32) so the shuffles see
// every lane.
__device__ __forceinline__ uint64_t warp_rounded(uint64_t n) { return (n + 31) & ~31ull; }

__device__ __forceinline__ void add_warp_sum(unsigned long long x, unsigned long long *counter) {
  for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(kFull, x, o);
  if ((threadIdx.x & 31) == 0 && x) atomicAdd(counter, x);
}

}  // namespace
}  // namespace mgb200

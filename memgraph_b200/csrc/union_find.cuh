// memgraph_b200/csrc/union_find.cuh -- the lock-free union-find shared by weakly connected components (wcc.cu),
// biconnectivity (biconnectivity.cu) and bipartite matching (bipartite_matching.cu): one uint32 parent per element.
// A link hooks the larger of two roots under the smaller one with atomicCAS and a compression only shortens paths, so
// parent[x] <= x always holds and every root is its set's smallest element, whatever order the threads link in.
#pragma once

#include <cstdint>

namespace mgb200 {
namespace {

__device__ __forceinline__ uint32_t load(const uint32_t *parent, uint32_t i) {
  return *(reinterpret_cast<const volatile uint32_t *>(parent) + i);  // other threads hook roots concurrently
}

// a[v] = v: every element its own set.
__global__ void __launch_bounds__(256) iota_kernel(uint64_t n, uint32_t *a) {
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n;
       v += static_cast<uint64_t>(gridDim.x) * blockDim.x)
    a[v] = static_cast<uint32_t>(v);
}

// Union of the sets of u and v: the larger root is hooked under the smaller one.
__device__ __forceinline__ void link(uint32_t u, uint32_t v, uint32_t *parent) {
  uint32_t p1 = load(parent, u), p2 = load(parent, v);
  while (p1 != p2) {
    const uint32_t high = max(p1, p2), low = min(p1, p2);
    const uint32_t p_high = load(parent, high);
    if (p_high == low) break;  // already hooked there
    if (p_high == high && atomicCAS(parent + high, high, low) == high) break;
    p1 = load(parent, load(parent, high));
    p2 = load(parent, low);
  }
}

// Every element points at its root afterwards.  Run only while no link is in flight.
__global__ void __launch_bounds__(256) compress_kernel(uint64_t n, uint32_t *parent) {
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n;
       v += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint32_t p0 = parent[v];
    uint32_t p = p0, pp = load(parent, p);
    while (p != pp) {
      p = pp;
      pp = load(parent, p);
    }
    if (p != p0) parent[v] = p;
  }
}

}  // namespace
}  // namespace mgb200

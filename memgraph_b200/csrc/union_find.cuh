// memgraph_b200/csrc/union_find.cuh -- the lock-free union-find shared by weakly connected components (wcc.cu),
// biconnectivity (biconnectivity.cu) and bipartite matching (bipartite_matching.cu): one uint32 parent per element.
// A link hooks the larger of two roots under the smaller one with atomicCAS and a compression only shortens paths, so
// parent[x] <= x always holds and every root is its set's smallest element, whatever order the threads link in.
// Also the numbering of such sets by their smallest member (number_sets), used by wcc.cu and strongly connected
// components (scc.cu).
#pragma once

#include <cuda_runtime.h>

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

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

struct IsRoot {
  const uint32_t *parent;
  __device__ __forceinline__ uint32_t operator()(uint64_t v) const { return parent[v] == v ? 1u : 0u; }
};

__global__ void __launch_bounds__(256) label_kernel(uint64_t n, const uint32_t *parent, const uint32_t *scan,
                                                    int64_t *component) {
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n;
       v += static_cast<uint64_t>(gridDim.x) * blockDim.x)
    component[v] = scan[parent[v]];
}

// component[v] = the rank of v's root among the roots, so sets are numbered in the order of their smallest member.
// Every element must point at its root (parent[v] == v for a root, parent[v] = its root otherwise); scan holds n
// values.  With tmp == nullptr only *tmp_bytes is set and nothing runs (CUB's size query); otherwise one exclusive scan
// of the root flags and one launch of label_kernel (a grid of `grid` blocks of 256 threads).
inline cudaError_t number_sets(uint64_t n, const uint32_t *parent, uint32_t *scan, int64_t *component, void *tmp,
                               size_t *tmp_bytes, int grid, cudaStream_t st) {
  const auto flags = thrust::make_transform_iterator(thrust::counting_iterator<uint64_t>(0), IsRoot{parent});
  const cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, *tmp_bytes, flags, scan, n, st);
  if (e != cudaSuccess || tmp == nullptr) return e;
  label_kernel<<<grid, 256, 0, st>>>(n, parent, scan, component);
  return cudaGetLastError();
}

}  // namespace
}  // namespace mgb200

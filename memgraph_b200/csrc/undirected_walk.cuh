// memgraph_b200/csrc/undirected_walk.cuh -- the entry walk over the undirected view of the BFS device graph and the
// breadth-first spanning forest built with it, shared by bridges / biconnected components (biconnectivity.cu) and
// maximum bipartite matching (bipartite_matching.cu).  Strongly connected components (scc.cu) walk directed lists with
// the same walk(): its scheduler only asks op.g.degree(u), so an op whose g is one direction's lists walks those.
//
// walk      an op visits the entries [rank, degree) of a vertex with stride `width`: a thread per vertex up to
//           kThreadEntries entries, a warp up to kWarpEntries and a block above, so hubs do not serialise a pass
// forest    a level-synchronous BFS from every root of a union-find (uf[v] == v) at once; the parent of a vertex is its
//           smallest-id neighbour in the previous level (atomicMin), so the forest does not depend on thread order.
//           Every level's vertices are kept (order[] + level offsets on the host), one host round trip per level
#pragma once

#include <cooperative_groups.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "bfs_graph.hpp"
#include "core.hpp"

namespace mgb200 {
namespace {

constexpr uint32_t kNone = 0xffffffffu;
constexpr uint64_t kThreadEntries = 16;  // entries a single thread walks
constexpr uint64_t kWarpEntries = 4096;  // above this, a block per vertex

struct Lists {  // the undirected view: out-list, then in-list
  const uint64_t *out_ptr;
  const uint32_t *out_adj;
  const uint64_t *in_ptr;
  const uint32_t *in_adj;
  __device__ __forceinline__ uint64_t degree(uint32_t u) const {
    return out_ptr[u + 1] - out_ptr[u] + in_ptr[u + 1] - in_ptr[u];
  }
};

struct Split {  // one entry-scan pass: vertices queued for a warp (front of the work list) or a block (back)
  unsigned int mid;
  unsigned int heavy;
  unsigned long long next;  // BFS: vertices appended to the next level
};

// Appends w to dst at a slot reserved with one atomic per group of converged threads.
__device__ __forceinline__ void append(uint32_t w, uint32_t *dst, unsigned long long *counter) {
  cooperative_groups::coalesced_group active = cooperative_groups::coalesced_threads();
  unsigned long long base = 0;
  if (active.thread_rank() == 0) base = atomicAdd(counter, static_cast<unsigned long long>(active.size()));
  base = active.shfl(base, 0);
  dst[base + active.thread_rank()] = w;
}

struct BfsOp {  // discovers the next level; the parent is the smallest frontier neighbour
  Lists g;
  int32_t *depth;
  uint32_t *tree_parent;
  uint32_t *next;  // order + end of the current level
  unsigned long long *next_count;
  int32_t next_depth;
  __device__ __forceinline__ void operator()(uint32_t u, uint64_t rank, uint64_t width) const {
    const uint64_t ob = g.out_ptr[u], od = g.out_ptr[u + 1] - ob;
    const uint64_t ib = g.in_ptr[u], id = g.in_ptr[u + 1] - ib;
    for (uint64_t i = rank; i < od + id; i += width) {
      const uint32_t w = i < od ? g.out_adj[ob + i] : g.in_adj[ib + (i - od)];
      int32_t d = *(reinterpret_cast<volatile int32_t *>(depth) + w);
      if (d == -1) {
        if (atomicCAS(depth + w, -1, next_depth) == -1) append(w, next, next_count);
        d = next_depth;  // whoever won set this level
      }
      if (d == next_depth) atomicMin(tree_parent + w, u);
    }
  }
};

// Items [lo, hi) of `items` (or the ids themselves when items is null): short lists walked by one thread, the others
// queued for walk_warp_kernel / walk_block_kernel.  Block 0 also clears `clear` for the next pass.
template <class Op>
__global__ void __launch_bounds__(kThreads) walk_thread_kernel(uint64_t lo, uint64_t hi, const uint32_t *items,
                                                               uint64_t n, Op op, uint32_t *work, Split *split,
                                                               Split *clear, unsigned long long *inspected) {
  if (clear && first_thread() == 0) *clear = Split{0, 0, 0};
  unsigned long long walked = 0;
  for (uint64_t i = lo + first_thread(); i < lo + warp_rounded(hi - lo); i += thread_count()) {
    if (i >= hi) continue;
    const uint32_t u = items ? items[i] : static_cast<uint32_t>(i);
    const uint64_t deg = op.g.degree(u);
    if (deg <= kThreadEntries) {
      op(u, 0, 1);
      walked += deg;
    } else if (deg <= kWarpEntries) {
      work[atomicAdd(&split->mid, 1u)] = u;
    } else {
      work[n - 1 - atomicAdd(&split->heavy, 1u)] = u;
    }
  }
  add_warp_sum(walked, inspected);
}

template <class Op>
__global__ void __launch_bounds__(kThreads) walk_warp_kernel(Op op, const uint32_t *work, const Split *split,
                                                             unsigned long long *inspected) {
  const uint32_t count = split->mid;
  const uint32_t lane = threadIdx.x & 31;
  unsigned long long walked = 0;
  for (uint64_t w = first_thread() >> 5; w < count; w += thread_count() >> 5) {
    const uint32_t u = work[w];
    op(u, lane, 32);
    if (lane == 0) walked += op.g.degree(u);
  }
  if (lane == 0 && walked) atomicAdd(inspected, walked);
}

template <class Op>
__global__ void __launch_bounds__(kThreads) walk_block_kernel(uint64_t n, Op op, const uint32_t *work,
                                                              const Split *split, unsigned long long *inspected) {
  const uint32_t count = split->heavy;
  unsigned long long walked = 0;
  for (uint32_t b = blockIdx.x; b < count; b += gridDim.x) {
    const uint32_t u = work[n - 1 - b];
    op(u, threadIdx.x, blockDim.x);
    if (threadIdx.x == 0) walked += op.g.degree(u);
  }
  if (threadIdx.x == 0 && walked) atomicAdd(inspected, walked);
}

// One entry-scan pass over items [lo, hi): thread, warp and block kernels.  `split` must be zero on entry; `clear`
// (may be null) is zeroed for the pass after this one.
template <class Op>
void walk(const mgb200_bfs_graph &g, uint64_t lo, uint64_t hi, const uint32_t *items, const Op &op, uint32_t *work,
          Split *split, Split *clear, unsigned long long *inspected, uint64_t *launches) {
  const uint64_t count = hi - lo;
  walk_thread_kernel<Op><<<blocks_for(count, g.sm_count, 8), kThreads, 0, g.stream>>>(lo, hi, items, g.n, op, work,
                                                                                      split, clear, inspected);
  walk_warp_kernel<Op><<<blocks_for(count * 32, g.sm_count, 16), kThreads, 0, g.stream>>>(op, work, split, inspected);
  walk_block_kernel<Op><<<static_cast<int>(std::min<uint64_t>(count, static_cast<uint64_t>(g.sm_count) * 8)), kThreads,
                          0, g.stream>>>(g.n, op, work, split, inspected);
  *launches += 3;
}

// Roots start level 0; every other vertex is undiscovered, its parent kNone until a frontier neighbour claims it.
// size (may be null) starts at 1 for every vertex.
__global__ void __launch_bounds__(kThreads) forest_init_kernel(uint64_t n, const uint32_t *uf, int32_t *depth,
                                                               uint32_t *tree_parent, uint32_t *size, uint32_t *order,
                                                               Split *split) {
  for (uint64_t v = first_thread(); v < n; v += thread_count()) {
    const bool root = uf[v] == v;
    depth[v] = root ? 0 : -1;
    tree_parent[v] = kNone;
    if (size) size[v] = 1;
    if (root) append(static_cast<uint32_t>(v), order, &split[1].next);  // level 0 clears it after the read
  }
}

// The forest from the roots of `uf` (compressed: every vertex points at its root) into g.depth, tree_parent and order:
// level L's vertices are order[(*level)[L], (*level)[L + 1]), and the last entry of *level closes an empty level.
// split[0..1] must be zero on entry; level L uses split[L & 1] and clears the other.
int bfs_forest(const mgb200_bfs_graph &g, const uint32_t *uf, uint32_t *tree_parent, uint32_t *size, uint32_t *order,
               uint32_t *work, Split *split, unsigned long long *inspected, std::vector<uint64_t> *level,
               uint64_t *launches) {
  cudaStream_t st = g.stream;
  const Lists lists{g.out_ptr, g.out_adj, g.in_ptr, g.in_adj};
  unsigned long long *host_next = g.host_counters;  // pinned
  forest_init_kernel<<<blocks_for(g.n, g.sm_count, 8), kThreads, 0, st>>>(g.n, uf, g.depth, tree_parent, size, order,
                                                                           split);
  ++*launches;
  level->assign(1, 0);
  MGB_CUDA(cudaMemcpyAsync(host_next, &split[1].next, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  level->push_back(*host_next);
  for (uint32_t L = 0;; ++L) {
    const uint64_t lo = (*level)[L], hi = (*level)[L + 1];
    if (lo == hi) break;
    // level L uses split[L & 1] and clears the other set, whose count the host has just read
    Split *cur = &split[L & 1], *clear = &split[(L + 1) & 1];
    const BfsOp op{lists, g.depth, tree_parent, order + hi, &cur->next, static_cast<int32_t>(L + 1)};
    walk(g, lo, hi, order, op, work, cur, clear, inspected, launches);
    MGB_CUDA(cudaMemcpyAsync(host_next, &cur->next, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    MGB_CUDA(cudaStreamSynchronize(st));
    level->push_back(hi + *host_next);
  }
  MGB_CUDA(cudaGetLastError());
  return MGB200_OK;
}

}  // namespace
}  // namespace mgb200

// memgraph_b200/csrc/betweenness.cu -- exact betweenness centrality (Brandes) for sm_90a (include/mgb200_bfs.h).
//
// Semantics: betweenness_centrality_alg::BetweennessCentrality, mage/cpp/betweenness_centrality_module/algorithm/
// betweenness_centrality.cpp:24-146 (restated and pinned in oracle/betweenness_oracle.c).
//
// Sources are processed in batches of S = 32, one warp lane per source, and every per-vertex quantity is stored
// vertex-major, [n][S]: an edge (u, v) then reads one contiguous row of u (256 B of sigma) instead of one scattered
// 8-byte value per source.
//   forward   level by level; every vertex with an undiscovered lane pulls sigma from its in-neighbours (both lists
//             when undirected) that are on the frontier in that lane.  fm[u] is the 32-bit mask of the lanes in which
//             u is at the current level: a neighbour whose mask misses the pending lanes is skipped without touching
//             its sigma row.  sigma is uint64_t and the adds are integer, so the sum is exact (modulo 2^64, as in the
//             reference) whatever the order.
//   backward  level by level from the deepest one, over the vertices discovered at that level (per-level vertex
//             lists written by the forward sweep): delta[v] = sigma[v] * sum over successors w one level deeper of
//             coef[w], coef[w] = (1 + delta[w]) / sigma[w].  coef replaces sigma[w] in place once w's level is done
//             (sigma[w] is not read again).  No float atomics: each (vertex, lane) is summed by one warp, in
//             adjacency order.
//   sum       bc[v] += delta (directed) or delta / 2 (undirected) for every lane that reached v at depth >= 1, added
//             one lane at a time in ascending source order -- the reference's order at threads = 1.
// A warp loads the rows of kLoadsInFlight candidate edges before it adds any, so the loads overlap.  Vertices whose
// pulled / pushed degree exceeds kHeavyDegree get a whole block, whose warps split the adjacency and
// combine their partial sums in warp order (deterministic).  Levels are launched kLevelsPerSync at a time before the
// host reads the frontier sizes; a level whose frontier is empty returns at once.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <new>
#include <vector>

#include "bfs_graph.hpp"
#include "core.hpp"
#include "mgb200_bfs.h"

namespace mgb200 {
namespace {

constexpr int S = MGB200_BC_BATCH;
constexpr int kWarps = kThreads / 32;
constexpr uint64_t kHeavyDegree = 512;  // above this, one block (8 warps) per vertex instead of one warp
constexpr int kLoadsInFlight = 8;        // candidate edges whose rows a warp loads before it adds any of them
constexpr int kLevelsPerSync = 8;
static_assert(S == 32, "one warp lane per source");

struct Lists {  // the adjacency a sweep walks: `a`, then `b` when undirected
  const uint64_t *a_ptr;
  const uint32_t *a_adj;
  const uint64_t *b_ptr;  // nullptr when directed
  const uint32_t *b_adj;
  __device__ __forceinline__ uint64_t degree(uint32_t v) const {
    uint64_t d = a_ptr[v + 1] - a_ptr[v];
    if (b_ptr) d += b_ptr[v + 1] - b_ptr[v];
    return d;
  }
};

struct State {                    // one batch; rows are [n][S]
  int32_t *depth;                 // valid only where the lane's bit of vis is set
  unsigned long long *sigma;      // sigma; after the backward sweep reached the lane's level: coef as double bits
  double *delta;
  uint32_t *vis;                  // [n] lanes that reached the vertex
  uint32_t *fm[2];                // [n] lanes for which the vertex is on the frontier, by level parity
  uint32_t *list;                 // vertices discovered per level, level L at [off[L], off[L] + cnt[L])
  unsigned long long *off;        // [levels]
  uint32_t *cnt;                  // [levels]
  unsigned long long *inspected;  // adjacency entries read
};

__device__ __forceinline__ uint64_t global_warp() {
  return (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
}
__device__ __forceinline__ uint64_t warp_count() { return (static_cast<uint64_t>(gridDim.x) * blockDim.x) >> 5; }

__global__ void init_batch_kernel(uint64_t n, uint64_t s0, uint32_t width, State st) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n; v += stride) {
    const bool source = v >= s0 && v < s0 + width;
    const uint32_t lane = static_cast<uint32_t>(v - s0);
    const uint32_t bit = source ? 1u << lane : 0u;
    st.vis[v] = bit;
    st.fm[0][v] = bit;
    if (source) {
      st.depth[v * S + lane] = 0;
      st.sigma[v * S + lane] = 1ull;
      st.list[lane] = static_cast<uint32_t>(v);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    st.off[0] = 0;
    st.cnt[0] = width;
    st.cnt[1] = 0;
  }
}

// Lanes `pend` of v pull sigma over one adjacency list; this warp reads chunks first, first + stride, ...
__device__ __forceinline__ void pull_sigma(const uint64_t *ptr, const uint32_t *adj, uint32_t v, uint64_t first,
                                           uint64_t stride, uint32_t pend, const uint32_t *fm,
                                           const unsigned long long *sigma, int lane, unsigned long long &acc,
                                           uint32_t &found, unsigned long long &inspected) {
  const uint64_t e = ptr[v + 1];
  for (uint64_t k = ptr[v] + first; k < e; k += stride) {
    uint32_t u = 0, mk = 0;
    if (k + lane < e) {
      u = adj[k + lane];
      mk = fm[u] & pend;
    }
    inspected += e - k < 32 ? e - k : 32;
    unsigned any = __ballot_sync(kFull, mk != 0);
    while (any) {  // kLoadsInFlight candidates at a time, so their loads overlap instead of waiting one by one
      uint32_t uj[kLoadsInFlight], mj[kLoadsInFlight];
      unsigned long long x[kLoadsInFlight];
#pragma unroll
      for (int q = 0; q < kLoadsInFlight; ++q) {
        const int j = any ? __ffs(any) - 1 : 0;
        const bool valid = any != 0;
        any &= any - 1;
        uj[q] = __shfl_sync(kFull, u, j);
        mj[q] = __shfl_sync(kFull, mk, j) & (valid ? kFull : 0u);
      }
#pragma unroll
      for (int q = 0; q < kLoadsInFlight; ++q)
        x[q] = ((mj[q] >> lane) & 1u) ? sigma[static_cast<uint64_t>(uj[q]) * S + lane] : 0ull;
#pragma unroll
      for (int q = 0; q < kLoadsInFlight; ++q) {
        acc += x[q];
        found |= mj[q];
      }
    }
  }
}

// The lanes of v found at level + 1: record sigma and depth, the next frontier mask and the level list.
__device__ __forceinline__ void discover(const State &st, uint32_t v, int lane, int level, uint32_t found,
                                         unsigned long long acc, uint64_t list_base, uint32_t *fm_next) {
  if (lane == 0) fm_next[v] = found;
  if (!found) return;
  if ((found >> lane) & 1u) {
    st.sigma[static_cast<uint64_t>(v) * S + lane] = acc;
    st.depth[static_cast<uint64_t>(v) * S + lane] = level + 1;
  }
  if (lane == 0) {
    st.vis[v] |= found;
    st.list[list_base + atomicAdd(st.cnt + level + 1, 1u)] = v;
  }
}

// Level `level` -> level + 1 for every vertex up to kHeavyDegree pulled edges: one warp per vertex.
__global__ void __launch_bounds__(kThreads) forward_kernel(uint64_t n, Lists pull, int level, uint32_t lane_mask,
                                                           State st) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    st.off[level + 1] = st.off[level] + st.cnt[level];
    st.cnt[level + 2] = 0;
  }
  if (st.cnt[level] == 0) return;  // the frontier is empty: the sweep has ended
  const int lane = threadIdx.x & 31;
  const uint32_t *fm = (level & 1) ? st.fm[1] : st.fm[0];  // a select, not a dynamic index (that would spill `st`)
  uint32_t *fm_next = (level & 1) ? st.fm[0] : st.fm[1];
  const uint64_t list_base = st.off[level] + st.cnt[level];
  unsigned long long inspected = 0;
  for (uint64_t w = global_warp(); w < n; w += warp_count()) {
    const uint32_t v = static_cast<uint32_t>(w);
    if (pull.degree(v) > kHeavyDegree) continue;
    const uint32_t pend = ~st.vis[v] & lane_mask;
    unsigned long long acc = 0;
    uint32_t found = 0;
    if (pend) {
      pull_sigma(pull.a_ptr, pull.a_adj, v, 0, 32, pend, fm, st.sigma, lane, acc, found, inspected);
      if (pull.b_ptr) pull_sigma(pull.b_ptr, pull.b_adj, v, 0, 32, pend, fm, st.sigma, lane, acc, found, inspected);
    }
    discover(st, v, lane, level, found, acc, list_base, fm_next);
  }
  if (lane == 0 && inspected) atomicAdd(st.inspected, inspected);
}

// The same for the vertices above kHeavyDegree: one block per vertex, the warps split the adjacency.
__global__ void __launch_bounds__(kThreads) forward_heavy_kernel(const uint32_t *heavy, uint32_t n_heavy, Lists pull,
                                                                 int level, uint32_t lane_mask, State st) {
  __shared__ unsigned long long s_acc[kWarps][S];
  __shared__ uint32_t s_found[kWarps];
  if (st.cnt[level] == 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t *fm = (level & 1) ? st.fm[1] : st.fm[0];
  uint32_t *fm_next = (level & 1) ? st.fm[0] : st.fm[1];
  const uint64_t list_base = st.off[level] + st.cnt[level];
  unsigned long long inspected = 0;
  for (uint32_t i = blockIdx.x; i < n_heavy; i += gridDim.x) {
    const uint32_t v = heavy[i];
    const uint32_t pend = ~st.vis[v] & lane_mask;
    unsigned long long acc = 0;
    uint32_t found = 0;
    if (pend) {
      pull_sigma(pull.a_ptr, pull.a_adj, v, warp * 32, kThreads, pend, fm, st.sigma, lane, acc, found, inspected);
      if (pull.b_ptr)
        pull_sigma(pull.b_ptr, pull.b_adj, v, warp * 32, kThreads, pend, fm, st.sigma, lane, acc, found, inspected);
    }
    s_acc[warp][lane] = acc;
    if (lane == 0) s_found[warp] = found;
    __syncthreads();
    if (warp == 0) {
      acc = 0;
      found = 0;
      for (int w = 0; w < kWarps; ++w) {
        acc += s_acc[w][lane];
        found |= s_found[w];
      }
      discover(st, v, lane, level, found, acc, list_base, fm_next);
    }
    __syncthreads();
  }
  if (lane == 0 && inspected) atomicAdd(st.inspected, inspected);
}

// Lanes `pend` of v (all at `level`) sum coef over the successors one level deeper, in adjacency order.
__device__ __forceinline__ void sum_coef(const uint64_t *ptr, const uint32_t *adj, uint32_t v, uint64_t first,
                                         uint64_t stride, uint32_t pend, int level, const State &st, int lane,
                                         double &s, unsigned long long &inspected) {
  const uint64_t e = ptr[v + 1];
  for (uint64_t k = ptr[v] + first; k < e; k += stride) {
    uint32_t x = 0, vx = 0;
    if (k + lane < e) {
      x = adj[k + lane];
      vx = st.vis[x] & pend;
    }
    inspected += e - k < 32 ? e - k : 32;
    unsigned any = __ballot_sync(kFull, vx != 0);
    while (any) {  // as in pull_sigma; the terms are still added in adjacency order
      uint64_t row[kLoadsInFlight];
      bool take[kLoadsInFlight];
      double term[kLoadsInFlight];
#pragma unroll
      for (int q = 0; q < kLoadsInFlight; ++q) {
        const int j = any ? __ffs(any) - 1 : 0;
        const bool valid = any != 0;
        any &= any - 1;
        row[q] = static_cast<uint64_t>(__shfl_sync(kFull, x, j)) * S + lane;
        take[q] = valid && ((__shfl_sync(kFull, vx, j) >> lane) & 1u);
      }
#pragma unroll
      for (int q = 0; q < kLoadsInFlight; ++q) take[q] = take[q] && st.depth[row[q]] == level + 1;
#pragma unroll
      for (int q = 0; q < kLoadsInFlight; ++q)
        term[q] = take[q] ? __longlong_as_double(static_cast<long long>(st.sigma[row[q]])) : 0.0;
#pragma unroll
      for (int q = 0; q < kLoadsInFlight; ++q)
        if (take[q]) s += term[q];
    }
  }
}

__device__ __forceinline__ uint32_t lanes_at(const State &st, uint32_t v, int lane, int level) {
  const uint64_t i = static_cast<uint64_t>(v) * S + lane;
  const bool mine = ((st.vis[v] >> lane) & 1u) && st.depth[i] == level;
  return __ballot_sync(kFull, mine);
}

// delta = sigma * s; sigma's slot becomes coef = (1 + delta) / sigma for the predecessors one level up.
__device__ __forceinline__ void settle(const State &st, uint32_t v, int lane, uint32_t pend, double s) {
  if (!((pend >> lane) & 1u)) return;
  const uint64_t i = static_cast<uint64_t>(v) * S + lane;
  const double sg = static_cast<double>(st.sigma[i]);
  const double d = sg * s;
  st.delta[i] = d;
  st.sigma[i] = static_cast<unsigned long long>(__double_as_longlong((1.0 + d) / sg));
}

__global__ void __launch_bounds__(kThreads) backward_kernel(const uint32_t *list, uint32_t count, Lists push, int level,
                                                            State st) {
  const int lane = threadIdx.x & 31;
  unsigned long long inspected = 0;
  for (uint64_t w = global_warp(); w < count; w += warp_count()) {
    const uint32_t v = list[w];
    if (push.degree(v) > kHeavyDegree) continue;
    const uint32_t pend = lanes_at(st, v, lane, level);
    if (!pend) continue;
    double s = 0.0;
    sum_coef(push.a_ptr, push.a_adj, v, 0, 32, pend, level, st, lane, s, inspected);
    if (push.b_ptr) sum_coef(push.b_ptr, push.b_adj, v, 0, 32, pend, level, st, lane, s, inspected);
    settle(st, v, lane, pend, s);
  }
  if (lane == 0 && inspected) atomicAdd(st.inspected, inspected);
}

__global__ void __launch_bounds__(kThreads) backward_heavy_kernel(const uint32_t *heavy, uint32_t n_heavy, Lists push,
                                                                  int level, State st) {
  __shared__ double s_part[kWarps][S];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long inspected = 0;
  for (uint32_t i = blockIdx.x; i < n_heavy; i += gridDim.x) {
    const uint32_t v = heavy[i];
    const uint32_t pend = lanes_at(st, v, lane, level);  // the same in every warp
    if (!pend) continue;
    double s = 0.0;
    sum_coef(push.a_ptr, push.a_adj, v, warp * 32, kThreads, pend, level, st, lane, s, inspected);
    if (push.b_ptr) sum_coef(push.b_ptr, push.b_adj, v, warp * 32, kThreads, pend, level, st, lane, s, inspected);
    s_part[warp][lane] = s;
    __syncthreads();
    if (warp == 0) {
      s = 0.0;
      for (int w = 0; w < kWarps; ++w) s += s_part[w][lane];
      settle(st, v, lane, pend, s);
    }
    __syncthreads();
  }
  if (lane == 0 && inspected) atomicAdd(st.inspected, inspected);
}

// bc[v] += delta (or delta / 2), lane by lane in ascending source order, for every lane that reached v at depth >= 1.
__global__ void __launch_bounds__(kThreads) accumulate_kernel(uint64_t n, int directed, State st, double *bc) {
  const int lane = threadIdx.x & 31;
  for (uint64_t w = global_warp(); w < n; w += warp_count()) {
    const uint32_t reached = st.vis[w];
    if (!reached) continue;
    const uint64_t i = w * S + lane;
    double value = 0.0;
    const bool on = ((reached >> lane) & 1u) && st.depth[i] >= 1;
    if (on) value = directed ? st.delta[i] : st.delta[i] / 2.0;
    unsigned lanes = __ballot_sync(kFull, on);
    if (!lanes) continue;
    double b = lane == 0 ? bc[w] : 0.0;
    while (lanes) {
      const int j = __ffs(lanes) - 1;
      lanes &= lanes - 1;
      const double x = __shfl_sync(kFull, value, j);
      if (lane == 0) b += x;
    }
    if (lane == 0) bc[w] = b;
  }
}

// vertices whose degree along `lists` exceeds kHeavyDegree
__global__ void heavy_list_kernel(uint64_t n, Lists lists, uint32_t *out, unsigned int *count) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n; v += stride)
    if (lists.degree(static_cast<uint32_t>(v)) > kHeavyDegree) out[atomicAdd(count, 1u)] = static_cast<uint32_t>(v);
}

}  // namespace
}  // namespace mgb200

using namespace mgb200;

extern "C" {

int mgb200_bc_run(mgb200_bfs_graph *g, int directed, uint64_t source_begin, uint64_t source_end,
                  int (*should_abort)(void *user), void *abort_user, double *bc_out, int bc_on_device,
                  mgb200_bc_stats *stats_out) {
  if (!g || source_begin > source_end || source_end > g->n || (g->n > 0 && !bc_out)) {
    set_error("betweenness: invalid argument (need 0 <= source_begin <= source_end <= n and a non-null bc_out)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  MGB_CUDA(cudaSetDevice(g->device));
  cudaStream_t st_ = g->stream;
  const uint64_t n = g->n;
  const Lists pull = directed ? Lists{g->in_ptr, g->in_adj, nullptr, nullptr}
                              : Lists{g->out_ptr, g->out_adj, g->in_ptr, g->in_adj};
  const Lists push = directed ? Lists{g->out_ptr, g->out_adj, nullptr, nullptr}
                              : Lists{g->out_ptr, g->out_adj, g->in_ptr, g->in_adj};
  const uint64_t max_levels = n + 2 * kLevelsPerSync + 4;
  mgb200_bc_stats stats{};
  stats.sources = source_end - source_begin;
  stats.batch_width = S;

  DeviceBuffers buf;
  State st{};
  double *bc = nullptr;
  uint32_t *heavy_pull = nullptr, *heavy_push = nullptr;
  unsigned int *heavy_count = nullptr;
  MGB_CUDA(buf.alloc(&st.depth, n * S));
  MGB_CUDA(buf.alloc(&st.sigma, n * S));
  MGB_CUDA(buf.alloc(&st.delta, n * S));
  MGB_CUDA(buf.alloc(&st.vis, n));
  MGB_CUDA(buf.alloc(&st.fm[0], n));
  MGB_CUDA(buf.alloc(&st.fm[1], n));
  MGB_CUDA(buf.alloc(&st.list, n * S));
  MGB_CUDA(buf.alloc(&st.off, max_levels));
  MGB_CUDA(buf.alloc(&st.cnt, max_levels));
  MGB_CUDA(buf.alloc(&st.inspected, 1));
  MGB_CUDA(buf.alloc(&bc, n));
  MGB_CUDA(buf.alloc(&heavy_pull, n));
  MGB_CUDA(buf.alloc(&heavy_push, n));
  MGB_CUDA(buf.alloc(&heavy_count, 2));
  unsigned long long *host_cnt = nullptr;  // pinned: the frontier sizes of one group of levels
  MGB_CUDA(cudaMallocHost(reinterpret_cast<void **>(&host_cnt), (kLevelsPerSync + 2) * sizeof(unsigned long long)));
  struct PinnedFree {
    void *p;
    ~PinnedFree() { cudaFreeHost(p); }
  } host_cnt_guard{host_cnt};
  uint32_t *level_cnt = reinterpret_cast<uint32_t *>(host_cnt);

  MGB_CUDA(cudaEventRecord(g->ev0, st_));
  MGB_CUDA(cudaMemsetAsync(bc, 0, std::max<uint64_t>(n, 1) * sizeof(double), st_));
  MGB_CUDA(cudaMemsetAsync(st.inspected, 0, sizeof(unsigned long long), st_));
  MGB_CUDA(cudaMemsetAsync(heavy_count, 0, 2 * sizeof(unsigned int), st_));
  if (n) {
    heavy_list_kernel<<<blocks_for(n, g->sm_count, 16), kThreads, 0, st_>>>(n, pull, heavy_pull, heavy_count);
    heavy_list_kernel<<<blocks_for(n, g->sm_count, 16), kThreads, 0, st_>>>(n, push, heavy_push, heavy_count + 1);
    stats.kernel_launches += 2;
  }
  unsigned int n_heavy[2] = {0, 0};
  MGB_CUDA(cudaMemcpyAsync(n_heavy, heavy_count, sizeof(n_heavy), cudaMemcpyDeviceToHost, st_));
  MGB_CUDA(cudaStreamSynchronize(st_));
  MGB_CUDA(cudaGetLastError());

  const int warp_grid = blocks_for(n * 32, g->sm_count, 8);
  std::vector<unsigned long long> off_host;
  std::vector<uint32_t> cnt_host;
  for (uint64_t s0 = source_begin; s0 < source_end; s0 += S) {
    if (should_abort && should_abort(abort_user)) {
      set_error("betweenness centrality: aborted by the caller");
      return MGB200_ERR_ABORTED;
    }
    const uint32_t width = static_cast<uint32_t>(std::min<uint64_t>(S, source_end - s0));
    const uint32_t lane_mask = width == 32 ? kFull : (1u << width) - 1u;
    init_batch_kernel<<<blocks_for(n, g->sm_count, 16), kThreads, 0, st_>>>(n, s0, width, st);
    stats.kernel_launches++;
    // forward: groups of levels, then one read of their frontier sizes
    int deepest = 0;
    for (int level = 0;; level += kLevelsPerSync) {
      for (int l = level; l < level + kLevelsPerSync; ++l) {
        forward_kernel<<<warp_grid, kThreads, 0, st_>>>(n, pull, l, lane_mask, st);
        stats.kernel_launches++;
        if (n_heavy[0]) {
          forward_heavy_kernel<<<std::min<unsigned>(n_heavy[0], g->sm_count * 8), kThreads, 0, st_>>>(
              heavy_pull, n_heavy[0], pull, l, lane_mask, st);
          stats.kernel_launches++;
        }
      }
      MGB_CUDA(cudaGetLastError());
      MGB_CUDA(cudaMemcpyAsync(level_cnt, st.cnt + level + 1, kLevelsPerSync * sizeof(uint32_t), cudaMemcpyDeviceToHost,
                               st_));
      MGB_CUDA(cudaStreamSynchronize(st_));
      int empty = -1;
      for (int l = 0; l < kLevelsPerSync && empty < 0; ++l)
        if (level_cnt[l] == 0) empty = l;
      if (empty >= 0) {
        deepest = level + empty;  // levels 0 .. deepest are non-empty
        break;
      }
      if (static_cast<uint64_t>(level + kLevelsPerSync) >= n) {  // cannot happen: a BFS has at most n levels
        set_error("betweenness: level count exceeded the vertex count");
        return MGB200_ERR_CUDA;
      }
    }
    stats.max_levels = std::max<uint32_t>(stats.max_levels, static_cast<uint32_t>(deepest));
    off_host.resize(deepest + 1);
    cnt_host.resize(deepest + 1);
    MGB_CUDA(cudaMemcpyAsync(off_host.data(), st.off, (deepest + 1) * sizeof(unsigned long long),
                             cudaMemcpyDeviceToHost, st_));
    MGB_CUDA(cudaMemcpyAsync(cnt_host.data(), st.cnt, (deepest + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, st_));
    MGB_CUDA(cudaStreamSynchronize(st_));
    // backward: deepest level first; the sources' own level 0 has no dependency to add
    for (int level = deepest; level >= 1; --level) {
      if (cnt_host[level]) {
        backward_kernel<<<blocks_for(static_cast<uint64_t>(cnt_host[level]) * 32, g->sm_count, 8), kThreads, 0, st_>>>(
            st.list + off_host[level], cnt_host[level], push, level, st);
        stats.kernel_launches++;
      }
      if (n_heavy[1]) {
        backward_heavy_kernel<<<std::min<unsigned>(n_heavy[1], g->sm_count * 8), kThreads, 0, st_>>>(
            heavy_push, n_heavy[1], push, level, st);
        stats.kernel_launches++;
      }
    }
    accumulate_kernel<<<warp_grid, kThreads, 0, st_>>>(n, directed, st, bc);
    stats.kernel_launches++;
    MGB_CUDA(cudaGetLastError());
    stats.batches++;
  }
  MGB_CUDA(cudaEventRecord(g->ev1, st_));
  unsigned long long inspected = 0;
  MGB_CUDA(cudaMemcpyAsync(&inspected, st.inspected, sizeof(inspected), cudaMemcpyDeviceToHost, st_));
  if (n)
    MGB_CUDA(cudaMemcpyAsync(bc_out, bc, n * sizeof(double),
                             bc_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st_));
  MGB_CUDA(cudaStreamSynchronize(st_));
  float ms = 0.f;
  MGB_CUDA(cudaEventElapsedTime(&ms, g->ev0, g->ev1));
  stats.edges_traversed = inspected;
  stats.run_ms = ms;
  if (stats_out) *stats_out = stats;
  return MGB200_OK;
}

int mgb200_betweenness_centrality(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, int directed,
                                  int normalized, double *bc_out) {
  if (n > 0 && !bc_out) {
    set_error("betweenness: bc_out is null");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  mgb200_bfs_graph *g = nullptr;
  int rc = mgb200_bfs_graph_create_host(0, n, m, from, to, &g);
  if (rc) return rc;
  rc = mgb200_bc_run(g, directed, 0, n, nullptr, nullptr, bc_out, 0, nullptr);
  mgb200_bfs_graph_destroy(g);
  if (rc) return rc;
  if (normalized) {  // betweenness_centrality.cpp:138-143; (n - 1) * (n - 2) in uint64_t
    const uint64_t pairs = (n - 1) * (n - 2);
    const double constant = n > 2 ? (directed ? 1.0 : 2.0) / static_cast<double>(pairs) : 1.0;
    for (uint64_t v = 0; v < n; ++v) bc_out[v] *= constant;
  }
  return MGB200_OK;
}

}  // extern "C"

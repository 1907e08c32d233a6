// memgraph_b200/csrc/bipartite_matching.cu -- maximum bipartite matching for sm_90a (include/mgb200_bfs.h).
//
// Semantics: the answer of the reference's bipartite_matching.max (mage/cpp/bipartite_matching_module; restated in
// oracle/bipartite_oracle.c): 0 when the undirected view has a self-loop or an odd cycle, otherwise the size of a
// maximum matching between the two colour classes.  The reference runs Kuhn's recursive DFS per left vertex; here the
// matching comes from alternating breadth-first searches (APFB, Deveci et al., "GPU accelerated maximum cardinality
// matching algorithms for bipartite graphs"), integer work only:
//   roots     union-find (union_find.cuh) over the undirected lists: every component's root is its smallest id
//   colour    undirected_walk.cuh's BFS forest from the roots; one pass over all entries flags (u, w) with
//             depth[u] == depth[w] (a self-loop included).  Anything flagged: not bipartite, nothing is matched.
//             Otherwise L = the even-depth vertices, R = the odd-depth ones
//   greedy    rounds while a round adds a pair, at most kGreedyRounds: every free L vertex proposes to its smallest free
//             neighbour, every R vertex accepts its smallest proposer (atomicMin)
//   phase     level 0 = the free L vertices, each the root of its own tree.  A level walks its L vertices' lists and
//             claims every unclaimed R neighbour once (BfsOp: pred[r] = the smallest frontier neighbour).  Then a free r
//             offers itself as its tree's end (end[root] = the smallest such r), and after that the mate of a matched r
//             joins the next level in the same tree, unless the tree has an end.  When no level is left, one thread per
//             tree with an end flips its path back to the root; trees are disjoint, so the paths are vertex-disjoint
//   stop      the first phase that finds no end.  By Berge's theorem the matching is then maximum, and with Z = the
//             vertices that search reached, (L \ Z) + (R n Z) is a vertex cover of its size (Konig's theorem)
// Every choice is a minimum over ids, so mate, cover and every stat but the time are the same from run to run.  Each
// search level costs a host round trip (the next level's size), as does each greedy round and each phase.
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

constexpr uint32_t kGreedyRounds = 4;

struct Counters {
  Split split[2];  // walk w uses split[w & 1] and clears the other for walk w + 1
  unsigned long long inspected;
  unsigned long long conflicts;  // entries (u, w) with depth[u] == depth[w]
  unsigned long long listed;     // L vertices in order[]: a greedy round's free ones, or a phase's search
  unsigned long long claimed;    // R vertices in rlist[]: those the phase's search claimed
  unsigned long long matched;    // pairs the greedy rounds made
  unsigned long long augmented;  // paths the phase flipped
  unsigned long long covered;    // vertices in the cover
};

__device__ __forceinline__ bool is_left(const int32_t *depth, uint32_t v) { return (depth[v] & 1) == 0; }

struct LinkOp {  // union-find over the entries
  Lists g;
  uint32_t *uf;
  __device__ __forceinline__ void operator()(uint32_t u, uint64_t rank, uint64_t width) const {
    const uint64_t ob = g.out_ptr[u], od = g.out_ptr[u + 1] - ob;
    const uint64_t ib = g.in_ptr[u], id = g.in_ptr[u + 1] - ib;
    for (uint64_t i = rank; i < od + id; i += width) link(u, i < od ? g.out_adj[ob + i] : g.in_adj[ib + (i - od)], uf);
  }
};

struct ConflictOp {  // counts the entries whose ends sit on the same forest level
  Lists g;
  const int32_t *depth;
  unsigned long long *conflicts;
  __device__ __forceinline__ void operator()(uint32_t u, uint64_t rank, uint64_t width) const {
    const uint64_t ob = g.out_ptr[u], od = g.out_ptr[u + 1] - ob;
    const uint64_t ib = g.in_ptr[u], id = g.in_ptr[u + 1] - ib;
    const int32_t du = depth[u];
    unsigned long long same = 0;
    for (uint64_t i = rank; i < od + id; i += width)
      same += depth[i < od ? g.out_adj[ob + i] : g.in_adj[ib + (i - od)]] == du;
    if (same) atomicAdd(conflicts, same);
  }
};

struct ProposeOp {  // target[u] = u's smallest free neighbour
  Lists g;
  const uint32_t *mate;
  uint32_t *target;
  __device__ __forceinline__ void operator()(uint32_t u, uint64_t rank, uint64_t width) const {
    const uint64_t ob = g.out_ptr[u], od = g.out_ptr[u + 1] - ob;
    const uint64_t ib = g.in_ptr[u], id = g.in_ptr[u + 1] - ib;
    uint32_t best = kNone;
    for (uint64_t i = rank; i < od + id; i += width) {
      const uint32_t w = i < od ? g.out_adj[ob + i] : g.in_adj[ib + (i - od)];
      if (mate[w] == kNone) best = min(best, w);
    }
    if (best != kNone) atomicMin(target + u, best);
  }
};

// The free L vertices into order[] (counted in `listed`).  With `search`, each becomes the root of its own tree for a
// phase: reached at level 0, no end yet.
__global__ void __launch_bounds__(kThreads) free_left_kernel(uint64_t n, const int32_t *depth, const uint32_t *mate,
                                                             bool search, uint32_t *tree, uint32_t *end,
                                                             int32_t *visit, uint32_t *order, Counters *counters) {
  for (uint64_t v = first_thread(); v < n; v += thread_count()) {
    const uint32_t u = static_cast<uint32_t>(v);
    if (!is_left(depth, u) || mate[u] != kNone) continue;
    if (search) {
      tree[u] = u;
      end[u] = kNone;
      visit[u] = 0;
    }
    append(u, order, &counters->listed);
  }
}

__global__ void __launch_bounds__(kThreads) accept_kernel(uint64_t count, const uint32_t *order,
                                                          const uint32_t *target, uint32_t *proposer) {
  for (uint64_t i = first_thread(); i < count; i += thread_count()) {
    const uint32_t u = order[i], t = target[u];
    if (t != kNone) atomicMin(proposer + t, u);
  }
}

__global__ void __launch_bounds__(kThreads) pair_kernel(uint64_t count, const uint32_t *order, const uint32_t *target,
                                                        const uint32_t *proposer, uint32_t *mate, Counters *counters) {
  unsigned long long made = 0;
  for (uint64_t i = first_thread(); i < warp_rounded(count); i += thread_count()) {
    if (i >= count) continue;
    const uint32_t u = order[i], t = target[u];
    if (t == kNone || proposer[t] != u) continue;
    mate[u] = t;
    mate[t] = u;
    ++made;
  }
  add_warp_sum(made, &counters->matched);
}

// The R vertices claimed at this level are rlist[lo, counters->claimed): a free one offers itself as its tree's end.
__global__ void __launch_bounds__(kThreads) settle_free_kernel(uint64_t lo, const uint32_t *rlist, const uint32_t *pred,
                                                               const uint32_t *tree, const uint32_t *mate,
                                                               uint32_t *end, const Counters *counters) {
  const uint64_t hi = counters->claimed;
  for (uint64_t i = lo + first_thread(); i < hi; i += thread_count()) {
    const uint32_t r = rlist[i];
    if (mate[r] == kNone) atomicMin(end + tree[pred[r]], r);
  }
}

// After settle_free_kernel: the mate of a matched one joins the next level in its tree, unless the tree has an end.
__global__ void __launch_bounds__(kThreads) settle_matched_kernel(uint64_t lo, const uint32_t *rlist,
                                                                  const uint32_t *pred, uint32_t *tree,
                                                                  const uint32_t *mate, const uint32_t *end,
                                                                  int32_t *visit, int32_t level, uint32_t *order,
                                                                  Counters *counters) {
  const uint64_t hi = counters->claimed;
  for (uint64_t i = lo + first_thread(); i < hi; i += thread_count()) {
    const uint32_t r = rlist[i], u = mate[r];
    if (u == kNone) continue;
    const uint32_t root = tree[pred[r]];
    if (end[root] != kNone) continue;
    tree[u] = root;
    visit[u] = level;
    append(u, order, &counters->listed);
  }
}

// One thread per tree with an end: flip the alternating path end -> root.
__global__ void __launch_bounds__(kThreads) augment_kernel(uint64_t roots, const uint32_t *order, const uint32_t *pred,
                                                           const uint32_t *end, uint32_t *mate, Counters *counters) {
  unsigned long long flipped = 0;
  for (uint64_t i = first_thread(); i < warp_rounded(roots); i += thread_count()) {
    if (i >= roots) continue;
    const uint32_t root = order[i];
    uint32_t r = end[root];
    if (r == kNone) continue;
    for (;;) {
      const uint32_t l = pred[r], next = mate[l];
      mate[r] = l;
      mate[l] = r;
      if (l == root) break;
      r = next;
    }
    ++flipped;
  }
  add_warp_sum(flipped, &counters->augmented);
}

// Konig's cover from the last (fruitless) search: L vertices it did not reach, R vertices it did.
__global__ void __launch_bounds__(kThreads) cover_kernel(uint64_t n, const int32_t *depth, const int32_t *visit,
                                                         uint8_t *cover, Counters *counters) {
  unsigned long long covered = 0;
  for (uint64_t v = first_thread(); v < warp_rounded(n); v += thread_count()) {
    if (v >= n) continue;
    const bool reached = visit[v] != -1;
    const bool in = is_left(depth, static_cast<uint32_t>(v)) ? !reached : reached;
    cover[v] = in ? 1 : 0;
    covered += in;
  }
  add_warp_sum(covered, &counters->covered);
}

}  // namespace
}  // namespace mgb200

using namespace mgb200;

extern "C" {

int mgb200_bipartite_matching_run(mgb200_bfs_graph *g, int (*should_abort)(void *user), void *abort_user,
                                  int64_t *mate_out, uint8_t *cover_out, mgb200_matching_stats *stats_out) {
  if (!g) {
    set_error("bipartite matching: invalid argument (need a graph)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  const uint64_t n = g->n;
  mgb200_matching_stats stats{};
  stats.bipartite = 1;
  if (n == 0) {
    if (stats_out) *stats_out = stats;
    return MGB200_OK;
  }
  MGB_CUDA(cudaSetDevice(g->device));
  cudaStream_t st = g->stream;
  const Lists lists{g->out_ptr, g->out_adj, g->in_ptr, g->in_adj};
  int32_t *depth = g->depth;
  uint32_t *order = g->queue[0], *work = g->queue[1];

  DeviceBuffers buf;
  uint32_t *tree = nullptr, *pred = nullptr, *mate = nullptr, *end = nullptr, *rlist = nullptr;
  int32_t *visit = nullptr;
  uint8_t *cover = nullptr;
  Counters *counters = nullptr;
  MGB_CUDA(buf.alloc(&tree, n));  // the union-find first, then a greedy round's targets, then each L vertex's tree
  MGB_CUDA(buf.alloc(&pred, n));  // the forest's parents first, then a greedy round's proposers, then each R's pred
  MGB_CUDA(buf.alloc(&mate, n));
  MGB_CUDA(buf.alloc(&end, n));
  MGB_CUDA(buf.alloc(&rlist, n));
  MGB_CUDA(buf.alloc(&visit, n));
  MGB_CUDA(buf.alloc(&cover, n));
  MGB_CUDA(buf.alloc(&counters, 1));

  const int grid_n = blocks_for(n, g->sm_count, 8);
  uint64_t launches = 0, walks = 0;
  auto run_walk = [&](uint64_t lo, uint64_t hi, const uint32_t *items, const auto &op) {
    walk(*g, lo, hi, items, op, work, &counters->split[walks & 1], &counters->split[(walks + 1) & 1],
         &counters->inspected, &launches);
    ++walks;
  };
  Counters host{};
  auto read = [&]() -> int {
    MGB_CUDA(cudaMemcpyAsync(&host, counters, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    MGB_CUDA(cudaStreamSynchronize(st));
    MGB_CUDA(cudaGetLastError());
    return MGB200_OK;
  };
  auto reset = [&](unsigned long long *counter) {
    return cudaMemsetAsync(counter, 0, sizeof(unsigned long long), st);
  };

  MGB_CUDA(cudaEventRecord(g->ev0, st));
  MGB_CUDA(cudaMemsetAsync(counters, 0, sizeof(Counters), st));

  // colouring: roots, the forest, then the same-level entries
  iota_kernel<<<grid_n, kThreads, 0, st>>>(n, tree);
  ++launches;
  run_walk(0, n, nullptr, LinkOp{lists, tree});
  compress_kernel<<<grid_n, kThreads, 0, st>>>(n, tree);
  ++launches;
  MGB_CUDA(cudaMemsetAsync(counters->split, 0, sizeof(counters->split), st));
  std::vector<uint64_t> level;
  int rc = bfs_forest(*g, tree, pred, nullptr, order, work, counters->split, &counters->inspected, &level, &launches);
  if (rc) return rc;
  MGB_CUDA(cudaMemsetAsync(counters->split, 0, sizeof(counters->split), st));
  walks = 0;
  run_walk(0, n, nullptr, ConflictOp{lists, depth, &counters->conflicts});
  if ((rc = read())) return rc;

  if (host.conflicts == 0) {
    // greedy rounds; the first listing is all of L, since nothing is matched yet
    MGB_CUDA(cudaMemsetAsync(mate, 0xff, n * sizeof(uint32_t), st));
    for (uint32_t round = 0;; ++round) {
      const unsigned long long before = host.matched;
      MGB_CUDA(reset(&counters->listed));
      free_left_kernel<<<grid_n, kThreads, 0, st>>>(n, depth, mate, false, tree, end, visit, order, counters);
      ++launches;
      if ((rc = read())) return rc;
      if (round == 0) stats.left_vertices = host.listed;
      if (host.listed == 0 || round == kGreedyRounds || (round > 0 && host.matched == before)) break;
      const uint64_t count = host.listed;
      MGB_CUDA(cudaMemsetAsync(tree, 0xff, n * sizeof(uint32_t), st));
      MGB_CUDA(cudaMemsetAsync(pred, 0xff, n * sizeof(uint32_t), st));
      run_walk(0, count, order, ProposeOp{lists, mate, tree});
      accept_kernel<<<blocks_for(count, g->sm_count, 8), kThreads, 0, st>>>(count, order, tree, pred);
      pair_kernel<<<blocks_for(count, g->sm_count, 8), kThreads, 0, st>>>(count, order, tree, pred, mate, counters);
      launches += 2;
    }
    stats.initial_matched = host.matched;
    stats.matched = host.matched;

    // phases until one finds no augmenting path
    for (;;) {
      if (should_abort && should_abort(abort_user) != 0) return set_error("procedure aborted by the host"), MGB200_ERR_ABORTED;
      ++stats.phases;
      MGB_CUDA(cudaMemsetAsync(visit, 0xff, n * sizeof(int32_t), st));
      MGB_CUDA(cudaMemsetAsync(pred, 0xff, n * sizeof(uint32_t), st));
      MGB_CUDA(reset(&counters->listed));
      MGB_CUDA(reset(&counters->claimed));
      MGB_CUDA(reset(&counters->augmented));
      free_left_kernel<<<grid_n, kThreads, 0, st>>>(n, depth, mate, true, tree, end, visit, order, counters);
      ++launches;
      if ((rc = read())) return rc;
      const uint64_t roots = host.listed;
      uint64_t lo = 0, hi = roots, r_lo = 0;
      uint32_t levels = 0;
      while (lo < hi) {
        ++levels;
        run_walk(lo, hi, order, BfsOp{lists, visit, pred, rlist, &counters->claimed, static_cast<int32_t>(levels)});
        const int grid_r = blocks_for(n - r_lo, g->sm_count, 8);
        settle_free_kernel<<<grid_r, kThreads, 0, st>>>(r_lo, rlist, pred, tree, mate, end, counters);
        settle_matched_kernel<<<grid_r, kThreads, 0, st>>>(r_lo, rlist, pred, tree, mate, end, visit,
                                                          static_cast<int32_t>(levels), order, counters);
        launches += 2;
        if ((rc = read())) return rc;
        r_lo = host.claimed;
        lo = hi;
        hi = host.listed;
      }
      stats.max_levels = std::max(stats.max_levels, levels);
      if (roots == 0) break;
      augment_kernel<<<blocks_for(roots, g->sm_count, 8), kThreads, 0, st>>>(roots, order, pred, end, mate, counters);
      ++launches;
      if ((rc = read())) return rc;
      if (host.augmented == 0) break;
      stats.matched += host.augmented;
    }
    cover_kernel<<<grid_n, kThreads, 0, st>>>(n, depth, visit, cover, counters);
    ++launches;
  } else {
    stats.bipartite = 0;
  }
  MGB_CUDA(cudaGetLastError());
  MGB_CUDA(cudaEventRecord(g->ev1, st));
  if ((rc = read())) return rc;
  float ms = 0.f;
  MGB_CUDA(cudaEventElapsedTime(&ms, g->ev0, g->ev1));

  if (mate_out || cover_out) {
    std::vector<uint32_t> mate_host(stats.bipartite ? n : 0);
    std::vector<uint8_t> cover_host(stats.bipartite ? n : 0);
    if (stats.bipartite) {
      MGB_CUDA(cudaMemcpyAsync(mate_host.data(), mate, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      MGB_CUDA(cudaMemcpyAsync(cover_host.data(), cover, n, cudaMemcpyDeviceToHost, st));
      MGB_CUDA(cudaStreamSynchronize(st));
    }
    for (uint64_t v = 0; v < n; ++v) {
      if (mate_out) mate_out[v] = stats.bipartite && mate_host[v] != kNone ? static_cast<int64_t>(mate_host[v]) : -1;
      if (cover_out) cover_out[v] = stats.bipartite ? cover_host[v] : 0;
    }
  }
  if (stats.bipartite && host.covered != stats.matched) {
    set_error("bipartite matching: the cover's size differs from the matching's (internal error)");
    return MGB200_ERR_CUDA;
  }
  stats.edges_inspected = host.inspected;
  stats.run_ms = ms;
  stats.kernel_launches = launches;
  if (stats_out) *stats_out = stats;
  return MGB200_OK;
}

int mgb200_maximum_bipartite_matching(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                      uint64_t *matched_out) {
  if (!matched_out) {
    set_error("bipartite matching: matched_out is null");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  mgb200_bfs_graph *g = nullptr;
  int rc = mgb200_bfs_graph_create_host(0, n, m, from, to, &g);
  if (rc) return rc;
  mgb200_matching_stats stats{};
  rc = mgb200_bipartite_matching_run(g, nullptr, nullptr, nullptr, nullptr, &stats);
  mgb200_bfs_graph_destroy(g);
  if (rc == MGB200_OK) *matched_out = stats.matched;
  return rc;
}

}  // extern "C"

// memgraph_b200/csrc/scc.cu -- strongly connected components for sm_90a (include/mgb200_bfs.h).
//
// Semantics: the partition of networkx.strongly_connected_components on the MultiDiGraph of all vertices and edges
// (the reference's nxalg.strongly_connected_components); self-loops and multi-edges change nothing.  component[v] is
// the rank of the smallest id of v's component among the components' smallest ids, as in wcc.cu.
//
// Multistep (Slota, Rajamanickam and Madduri, IPDPS 2014), made deterministic; integer work only.  Every vertex is
// live until its representative rep[v] (the smallest id of its component) is set:
//   trim      live in- and out-counts (entries w == v not counted).  A vertex with a zero count is a singleton
//             component: it is peeled, and peeling walks its lists and decrements its neighbours' counts.  The thread
//             that drives a count to zero claims the neighbour (atomicCAS on rep) and, if its list is short
//             (kThreadEntries), peels it at once: it follows one such claim itself and queues the others on a spill
//             list that drain_kernel empties in the same level.  Longer lists wait for the next level.  A path is
//             therefore trimmed in one level; the peeled set is the unique fixed point, so thread order cannot change it
//   pivot     the live vertex with the largest in_count * out_count (ties: the smaller id).  A forward search over
//             live out-lists, then a backward search over in-lists restricted to what the forward search reached: the
//             vertices both reached are the pivot's component, represented by their smallest id
//   colour    while a vertex is live: colour[v] = v, the minimum is propagated forward over live out-edges until
//             nothing changes; every v with colour[v] == v is a root and the smallest id of its component, which a
//             multi-source backward search over in-edges between vertices of the same colour collects.  A level
//             propagates the colours its frontier held when it started (snap[], written before the level's walk), so
//             which vertices a level lowers does not depend on thread order
//   number    union_find.cuh's numbering of sets by their smallest member
// Every search runs level by level through one frontier driver: a level of more than kNarrow vertices is one walk()
// of undirected_walk.cuh (thread / warp / block per list, one host round trip); from kNarrow vertices down, one CTA
// expands up to kNarrowLevels levels in one launch, with block barriers between them.  The frontiers, and with them
// every stat but the time, are the same from run to run.
#include <cooperative_groups.h>
#include <cooperative_groups/reduce.h>

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include <algorithm>
#include <cstdint>

#include "bfs_graph.hpp"
#include "core.hpp"
#include "mgb200_bfs.h"
#include "undirected_walk.cuh"
#include "union_find.cuh"

namespace mgb200 {
namespace {

constexpr int kNarrowThreads = 256;
constexpr uint32_t kNarrowItems = 4;                         // frontier vertices per thread of the narrow CTA
constexpr uint64_t kNarrow = kNarrowThreads * kNarrowItems;  // largest frontier the narrow CTA expands
constexpr uint32_t kNarrowLevels = 1024;                     // levels per narrow launch, then the host polls again

struct Narrow {  // what a narrow launch hands back
  unsigned long long count;    // the frontier it stopped at
  unsigned long long reached;  // vertices its levels appended
  unsigned int cur;            // the queue holding that frontier
  unsigned int levels;
};

struct Counters {
  Split split[2];                  // walk w uses split[w & 1] and clears the other for walk w + 1
  unsigned long long inspected;
  unsigned long long next;         // vertices appended to the next frontier (a wide level, a trim level)
  unsigned long long listed;       // trim seeds, colouring roots
  unsigned long long trimmed;      // claims of the trim
  unsigned long long spill_head;   // the trim's spill list: [spill_head, spill_tail) still to be peeled
  unsigned long long spill_tail;
  unsigned long long pivot_size;
  uint32_t pivot_rep;
  uint32_t pad;
  Narrow narrow;
};

__device__ __forceinline__ uint32_t vload(const uint32_t *a, uint64_t i) {
  return *(reinterpret_cast<const volatile uint32_t *>(a) + i);  // written by other threads of the same launch
}

struct DirList {  // one direction of the device graph: the out-lists (CSR) or the in-lists (CSC)
  const uint64_t *ptr;
  const uint32_t *adj;
  __device__ __forceinline__ uint64_t degree(uint32_t u) const { return ptr[u + 1] - ptr[u]; }
  __device__ __forceinline__ uint32_t entry(uint32_t u, uint64_t i) const { return adj[ptr[u] + i]; }
};

// An op walked by walk() (operator()) and by narrow_kernel (visit): entry i of u's list.  prepare(u) runs for every
// frontier vertex before the level's walk (a separate launch for a wide level, only where kSnapshot<Op>).
template <class Derived>
struct EntryOp {
  __device__ __forceinline__ void prepare(uint32_t) const {}
  __device__ __forceinline__ void operator()(uint32_t u, uint64_t rank, uint64_t width) const {
    const Derived &op = static_cast<const Derived &>(*this);
    const uint64_t d = op.g.degree(u);
    for (uint64_t i = rank; i < d; i += width) op.visit(u, i);
  }
};

struct ForwardOp : EntryOp<ForwardOp> {  // live out-neighbours: mark 0 -> 1
  DirList g;
  const uint32_t *rep;
  uint32_t *mark;
  uint32_t *next;
  unsigned long long *next_count;
  uint32_t stamp;
  __device__ __forceinline__ void visit(uint32_t u, uint64_t i) const {
    const uint32_t w = g.entry(u, i);
    if (rep[w] == kNone && vload(mark, w) == 0 && atomicCAS(mark + w, 0u, 1u) == 0u) append(w, next, next_count);
  }
};

struct BackwardOp : EntryOp<BackwardOp> {  // in-neighbours the forward search reached: mark 1 -> 2, smallest id kept
  DirList g;
  uint32_t *mark;
  uint32_t *smallest;
  uint32_t *next;
  unsigned long long *next_count;
  uint32_t stamp;
  __device__ __forceinline__ void visit(uint32_t u, uint64_t i) const {
    const uint32_t w = g.entry(u, i);
    if (vload(mark, w) != 1 || atomicCAS(mark + w, 1u, 2u) != 1u) return;
    append(w, next, next_count);
    cooperative_groups::coalesced_group active = cooperative_groups::coalesced_threads();
    const uint32_t low = cooperative_groups::reduce(active, w, cooperative_groups::less<uint32_t>());
    if (active.thread_rank() == 0) atomicMin(smallest, low);
  }
};

struct PropagateOp : EntryOp<PropagateOp> {  // live out-neighbours take the snapshot colour if it is smaller
  DirList g;
  const uint32_t *rep;
  uint32_t *colour;
  uint32_t *snap;
  uint32_t *queued;  // the stamp of the last level that appended the vertex
  uint32_t *next;
  unsigned long long *next_count;
  uint32_t stamp;
  __device__ __forceinline__ void prepare(uint32_t u) const { snap[u] = vload(colour, u); }
  __device__ __forceinline__ void visit(uint32_t u, uint64_t i) const {
    const uint32_t w = g.entry(u, i), c = snap[u];
    if (rep[w] != kNone || vload(colour, w) <= c) return;
    if (atomicMin(colour + w, c) > c && atomicExch(queued + w, stamp) != stamp) append(w, next, next_count);
  }
};

template <class Op>
constexpr bool kSnapshot = false;
template <>
constexpr bool kSnapshot<PropagateOp> = true;

struct CollectOp : EntryOp<CollectOp> {  // live in-neighbours of the same colour join the root's component
  DirList g;
  const uint32_t *colour;
  uint32_t *rep;
  uint32_t *next;
  unsigned long long *next_count;
  uint32_t stamp;
  __device__ __forceinline__ void visit(uint32_t u, uint64_t i) const {
    const uint32_t w = g.entry(u, i), c = colour[u];
    if (colour[w] == c && vload(rep, w) == kNone && atomicCAS(rep + w, kNone, c) == kNone) append(w, next, next_count);
  }
};

struct TrimOp {  // peels a vertex: walks both lists (Lists: out-list, then in-list) and decrements the counts
  Lists g;
  uint32_t *in_count;
  uint32_t *out_count;
  uint32_t *rep;
  uint32_t *next;  // long lists claimed: the next level
  unsigned long long *next_count;
  uint32_t *spill;  // short lists claimed beyond the one a thread follows
  unsigned long long *spill_tail;
  unsigned long long *trimmed;
  unsigned long long *inspected;

  // Entries [rank, degree) of u with stride width.  Returns `follow`, or the first short claim if follow is kNone.
  __device__ __forceinline__ uint32_t peel(uint32_t u, uint64_t rank, uint64_t width, uint32_t follow) const {
    const uint64_t ob = g.out_ptr[u], od = g.out_ptr[u + 1] - ob;
    const uint64_t ib = g.in_ptr[u], id = g.in_ptr[u + 1] - ib;
    unsigned long long claimed = 0;
    for (uint64_t i = rank; i < od + id; i += width) {
      const bool out = i < od;
      const uint32_t w = out ? g.out_adj[ob + i] : g.in_adj[ib + (i - od)];
      if (w == u || vload(rep, w) != kNone) continue;
      // an out-entry u -> w loses w an in-entry, an in-entry w -> u loses w an out-entry
      if (atomicSub(out ? in_count + w : out_count + w, 1u) != 1u) continue;
      if (atomicCAS(rep + w, kNone, w) != kNone) continue;  // its other count reached zero first
      ++claimed;
      if (g.degree(w) > kThreadEntries) {
        append(w, next, next_count);
      } else if (follow == kNone) {
        follow = w;
      } else {
        append(w, spill, spill_tail);
      }
    }
    if (claimed) atomicAdd(trimmed, claimed);
    return follow;
  }

  // Peels the chain of short claims that starts at x.
  __device__ __forceinline__ void chain(uint32_t x) const {
    unsigned long long walked = 0;
    while (x != kNone) {
      walked += g.degree(x);
      x = peel(x, 0, 1, kNone);
    }
    if (walked) atomicAdd(inspected, walked);
  }

  __device__ __forceinline__ void operator()(uint32_t u, uint64_t rank, uint64_t width) const {
    chain(peel(u, rank, width, kNone));
  }
};

// Live counts; a vertex with a zero count is trimmed at once and seeds level 0 (order[], counted in `listed`).
__device__ __forceinline__ uint64_t copies(const uint32_t *adj, uint64_t lo, uint64_t hi, uint32_t v) {
  uint64_t a = lo, b = hi;  // lower bound of v in the sorted row
  while (a < b) {
    const uint64_t mid = (a + b) / 2;
    if (adj[mid] < v) a = mid + 1; else b = mid;
  }
  uint64_t e = a;
  while (e < hi && adj[e] == v) ++e;
  return e - a;
}

__global__ void __launch_bounds__(kThreads) trim_init_kernel(uint64_t n, Lists g, uint32_t *in_count,
                                                             uint32_t *out_count, uint32_t *rep, uint32_t *order,
                                                             Counters *counters) {
  for (uint64_t v = first_thread(); v < n; v += thread_count()) {
    const uint32_t u = static_cast<uint32_t>(v);
    const uint64_t ob = g.out_ptr[v], oe = g.out_ptr[v + 1], ib = g.in_ptr[v], ie = g.in_ptr[v + 1];
    const uint32_t out = static_cast<uint32_t>(oe - ob - copies(g.out_adj, ob, oe, u));
    const uint32_t in = static_cast<uint32_t>(ie - ib - copies(g.in_adj, ib, ie, u));
    in_count[v] = in;
    out_count[v] = out;
    const bool trimmed = in == 0 || out == 0;
    rep[v] = trimmed ? u : kNone;
    if (trimmed) append(u, order, &counters->listed);
  }
}

// The spill list of a trim level: a thread takes the next entry, peels it and its chain, until the list is empty.  A
// thread that spills an entry is still working, so it finds the entry here if nobody took it first.
__global__ void __launch_bounds__(kThreads) drain_kernel(TrimOp op, const uint32_t *spill, Counters *counters) {
  volatile unsigned long long *head = &counters->spill_head, *tail = &counters->spill_tail;
  for (;;) {
    const unsigned long long h = *head;
    if (h >= *tail) return;
    if (atomicCAS(&counters->spill_head, h, h + 1) != h) continue;
    uint32_t x;
    while ((x = vload(spill, h)) == kNone) {  // reserved, the store is on its way
    }
    op.chain(x);
  }
}

struct PivotKey {  // in_count * out_count of a live vertex, 0 for the others
  const uint32_t *rep, *in_count, *out_count;
  __device__ __forceinline__ uint64_t operator()(uint64_t v) const {
    return rep[v] == kNone ? static_cast<uint64_t>(in_count[v]) * out_count[v] : 0;
  }
};

// The pivot alone in the first frontier of a search; `reached` is its mark (1 forward, 2 backward).
__global__ void seed_kernel(const int64_t *pivot, uint32_t reached, uint32_t *mark, uint32_t *queue,
                            Counters *counters) {
  const uint32_t p = static_cast<uint32_t>(*pivot);
  mark[p] = reached;
  queue[0] = p;
  counters->pivot_rep = p;
}

// The pivot's component (mark == 2) gets its smallest id as representative.
__global__ void __launch_bounds__(kThreads) pivot_component_kernel(uint64_t n, uint32_t *mark, uint32_t *rep,
                                                                   Counters *counters) {
  const uint32_t low = counters->pivot_rep;
  unsigned long long mine = 0;
  for (uint64_t v = first_thread(); v < warp_rounded(n); v += thread_count()) {
    if (v >= n || mark[v] != 2) continue;
    rep[v] = low;
    ++mine;
  }
  add_warp_sum(mine, &counters->pivot_size);
}

// A colouring round starts: every live vertex has its own id as colour and is in the first frontier.
__global__ void __launch_bounds__(kThreads) colour_init_kernel(uint64_t n, const uint32_t *rep, uint32_t *colour,
                                                               uint32_t *queue, Counters *counters) {
  for (uint64_t v = first_thread(); v < n; v += thread_count()) {
    if (rep[v] != kNone) continue;
    colour[v] = static_cast<uint32_t>(v);
    append(static_cast<uint32_t>(v), queue, &counters->next);
  }
}

// Live vertices that kept their own colour are roots: their own representatives and the backward searches' sources.
__global__ void __launch_bounds__(kThreads) roots_kernel(uint64_t n, const uint32_t *colour, uint32_t *rep,
                                                         uint32_t *queue, Counters *counters) {
  for (uint64_t v = first_thread(); v < n; v += thread_count()) {
    if (rep[v] != kNone || colour[v] != v) continue;
    rep[v] = static_cast<uint32_t>(v);
    append(static_cast<uint32_t>(v), queue, &counters->listed);
  }
}

template <class Op>
__global__ void __launch_bounds__(kThreads) prepare_kernel(uint64_t count, const uint32_t *items, Op op) {
  for (uint64_t i = first_thread(); i < count; i += thread_count()) op.prepare(items[i]);
}

// Up to kNarrowLevels levels from a frontier of at most kNarrow vertices, in one CTA: the frontier's lists are dealt
// out entry by entry (a block scan of the degrees, then a binary search per entry), so a hub in a narrow frontier is
// walked by every thread.  Stops when the frontier empties or outgrows kNarrow.
template <class Op>
__global__ void __launch_bounds__(kNarrowThreads) narrow_kernel(Op op, uint32_t *q0, uint32_t *q1, uint32_t cur,
                                                                unsigned long long count, Counters *counters) {
  using Scan = cub::BlockScan<unsigned long long, kNarrowThreads>;
  __shared__ typename Scan::TempStorage scan_storage;
  __shared__ unsigned long long start[kNarrow + 1];
  __shared__ uint32_t front[kNarrow];
  volatile unsigned long long *next_count = op.next_count;
  const uint32_t first_stamp = op.stamp;
  uint32_t levels = 0;
  unsigned long long reached = 0, walked = 0;
  while (count > 0 && count <= kNarrow && levels < kNarrowLevels) {
    const uint32_t *items = cur ? q1 : q0;
    unsigned long long deg[kNarrowItems];
    for (uint32_t k = 0; k < kNarrowItems; ++k) {
      const uint64_t i = threadIdx.x * kNarrowItems + k;
      deg[k] = 0;
      if (i < count) {
        const uint32_t u = items[i];
        front[i] = u;
        deg[k] = op.g.degree(u);
        op.prepare(u);
      }
    }
    unsigned long long total = 0;
    Scan(scan_storage).ExclusiveSum(deg, deg, total);
    for (uint32_t k = 0; k < kNarrowItems; ++k) {
      const uint64_t i = threadIdx.x * kNarrowItems + k;
      if (i < count) start[i] = deg[k];
    }
    if (threadIdx.x == 0) {
      start[count] = total;
      *next_count = 0;
    }
    op.next = cur ? q0 : q1;
    op.stamp = first_stamp + levels;
    __syncthreads();
    uint32_t k = 0;  // the frontier vertex holding entry j: start[k] <= j < start[k + 1]; j only grows
    for (unsigned long long j = threadIdx.x; j < total; j += kNarrowThreads) {
      uint32_t hi = static_cast<uint32_t>(count);
      while (hi - k > 1) {
        const uint32_t mid = (k + hi) / 2;
        if (start[mid] <= j) k = mid; else hi = mid;
      }
      op.visit(front[k], j - start[k]);
    }
    walked += total;
    __syncthreads();
    count = *next_count;
    reached += count;
    cur ^= 1;
    ++levels;
    __syncthreads();  // every thread has read the count before thread 0 clears it
  }
  if (threadIdx.x == 0) {
    counters->narrow = Narrow{count, reached, cur, levels};
    if (walked) atomicAdd(&counters->inspected, walked);
  }
}

// size[rep] += members; the lanes of a warp with the same representative add once.
__global__ void __launch_bounds__(kThreads) size_kernel(uint64_t n, const uint32_t *rep, uint32_t *size) {
  for (uint64_t v = first_thread(); v < warp_rounded(n); v += thread_count()) {
    const uint32_t r = v < n ? rep[v] : kNone;
    const unsigned peers = __match_any_sync(kFull, r);
    if (r != kNone && (threadIdx.x & 31) == static_cast<unsigned>(__ffs(peers) - 1)) atomicAdd(size + r, __popc(peers));
  }
}

// One call's device state and the frontier driver shared by the searches and the propagation.
struct Run {
  const mgb200_bfs_graph &g;
  int (*should_abort)(void *);
  void *abort_user;
  Counters *counters;
  uint32_t *queue[2];
  uint32_t *work;
  mgb200_scc_stats &stats;
  Counters host{};
  uint64_t walks = 0;
  uint32_t stamp = 0;

  int fetch() {
    MGB_CUDA(cudaMemcpyAsync(&host, counters, sizeof(Counters), cudaMemcpyDeviceToHost, g.stream));
    MGB_CUDA(cudaStreamSynchronize(g.stream));
    MGB_CUDA(cudaGetLastError());
    return MGB200_OK;
  }
  int read() {  // a round trip of the run: the host waits for the device to decide what to launch next
    ++stats.host_round_trips;
    return fetch();
  }

  int poll() const {
    if (should_abort && should_abort(abort_user) != 0) return set_error("procedure aborted by the host"), MGB200_ERR_ABORTED;
    return MGB200_OK;
  }

  template <class Op>
  void walk_level(uint64_t lo, uint64_t hi, const uint32_t *items, const Op &op) {
    walk(g, lo, hi, items, op, work, &counters->split[walks & 1], &counters->split[(walks + 1) & 1],
         &counters->inspected, &stats.kernel_launches);
    ++walks;
  }

  // Levels from the frontier queue[cur][0, count) until it is empty; *reached = the vertices appended.
  template <class Op>
  int frontier(Op op, uint32_t cur, uint64_t count, uint64_t *reached) {
    cudaStream_t st = g.stream;
    op.next_count = &counters->next;
    *reached = 0;
    while (count > 0) {
      if (int rc = poll()) return rc;
      if (count <= kNarrow) {
        op.stamp = stamp + 1;
        narrow_kernel<Op><<<1, kNarrowThreads, 0, st>>>(op, queue[0], queue[1], cur, count, counters);
        ++stats.kernel_launches;
        if (int rc = read()) return rc;
        count = host.narrow.count;
        cur = host.narrow.cur;
        *reached += host.narrow.reached;
        stats.levels += host.narrow.levels;
        stamp += host.narrow.levels;
      } else {
        op.next = queue[cur ^ 1];
        op.stamp = ++stamp;
        MGB_CUDA(cudaMemsetAsync(&counters->next, 0, sizeof(unsigned long long), st));
        if constexpr (kSnapshot<Op>) {
          prepare_kernel<Op><<<blocks_for(count, g.sm_count, 8), kThreads, 0, st>>>(count, queue[cur], op);
          ++stats.kernel_launches;
        }
        walk_level(0, count, queue[cur], op);
        if (int rc = read()) return rc;
        count = host.next;
        cur ^= 1;
        *reached += count;
        ++stats.levels;
      }
    }
    return MGB200_OK;
  }
};

}  // namespace
}  // namespace mgb200

using namespace mgb200;

extern "C" {

int mgb200_scc_run(mgb200_bfs_graph *g, int (*should_abort)(void *user), void *abort_user, int64_t *component_out,
                   mgb200_scc_stats *stats_out) {
  if (!g || (g->n > 0 && !component_out)) {
    set_error("strongly connected components: invalid argument (need a graph and a non-null component_out)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  mgb200_scc_stats stats{};
  const uint64_t n = g->n;
  if (n == 0) {
    if (stats_out) *stats_out = stats;
    return MGB200_OK;
  }
  MGB_CUDA(cudaSetDevice(g->device));
  cudaStream_t st = g->stream;
  const Lists lists{g->out_ptr, g->out_adj, g->in_ptr, g->in_adj};
  const DirList out{g->out_ptr, g->out_adj}, in{g->in_ptr, g->in_adj};

  DeviceBuffers buf;
  uint32_t *rep = nullptr, *in_count = nullptr, *out_count = nullptr, *mark = nullptr, *colour = nullptr,
           *snap = nullptr, *queued = nullptr, *q0 = nullptr, *q1 = nullptr, *work = nullptr, *size = nullptr,
           *scan = nullptr, *largest = nullptr;
  int64_t *component = nullptr, *pivot = nullptr;
  uint64_t *pivot_key = nullptr;
  Counters *counters = nullptr;
  MGB_CUDA(buf.alloc(&rep, n));
  MGB_CUDA(buf.alloc(&in_count, n));
  MGB_CUDA(buf.alloc(&out_count, n));
  MGB_CUDA(buf.alloc(&mark, n));
  MGB_CUDA(buf.alloc(&colour, n));
  MGB_CUDA(buf.alloc(&snap, n));
  MGB_CUDA(buf.alloc(&queued, n));
  MGB_CUDA(buf.alloc(&q0, n));  // the trim's order first, then a frontier queue
  MGB_CUDA(buf.alloc(&q1, n));  // the trim's spill list first, then a frontier queue
  MGB_CUDA(buf.alloc(&work, n));
  MGB_CUDA(buf.alloc(&size, n));
  MGB_CUDA(buf.alloc(&scan, n));
  MGB_CUDA(buf.alloc(&largest, 1));
  MGB_CUDA(buf.alloc(&component, n));
  MGB_CUDA(buf.alloc(&pivot, 1));
  MGB_CUDA(buf.alloc(&pivot_key, 1));
  MGB_CUDA(buf.alloc(&counters, 1));
  const auto keys = thrust::make_transform_iterator(thrust::counting_iterator<uint64_t>(0),
                                                    PivotKey{rep, in_count, out_count});
  size_t argmax_bytes = 0, max_bytes = 0, number_bytes = 0;
  MGB_CUDA(cub::DeviceReduce::ArgMax(nullptr, argmax_bytes, keys, pivot_key, pivot, static_cast<int64_t>(n), st));
  MGB_CUDA(cub::DeviceReduce::Max(nullptr, max_bytes, size, largest, n, st));
  MGB_CUDA(number_sets(n, rep, scan, component, nullptr, &number_bytes, 1, st));
  char *cub_tmp = nullptr;
  const size_t cub_bytes = std::max(argmax_bytes, std::max(max_bytes, number_bytes));
  MGB_CUDA(buf.alloc(&cub_tmp, cub_bytes));

  Run run{*g, should_abort, abort_user, counters, {q0, q1}, work, stats};
  const int grid = blocks_for(n, g->sm_count, 8);
  int rc = MGB200_OK;
  MGB_CUDA(cudaEventRecord(g->ev0, st));
  MGB_CUDA(cudaMemsetAsync(counters, 0, sizeof(Counters), st));
  MGB_CUDA(cudaMemsetAsync(mark, 0, n * sizeof(uint32_t), st));
  MGB_CUDA(cudaMemsetAsync(queued, 0, n * sizeof(uint32_t), st));
  MGB_CUDA(cudaMemsetAsync(size, 0, n * sizeof(uint32_t), st));
  MGB_CUDA(cudaMemsetAsync(q1, 0xff, n * sizeof(uint32_t), st));

  // trim: level L walks order[lo, hi) and its spill list; its long claims are order[hi, ...)
  trim_init_kernel<<<grid, kThreads, 0, st>>>(n, lists, in_count, out_count, rep, q0, counters);
  ++stats.kernel_launches;
  if ((rc = run.read())) return rc;
  uint64_t lo = 0, hi = run.host.listed;
  while (lo < hi) {
    if ((rc = run.poll())) return rc;
    const TrimOp op{lists,  in_count, out_count, rep, q0 + hi, &counters->next, q1, &counters->spill_tail,
                    &counters->trimmed, &counters->inspected};
    MGB_CUDA(cudaMemsetAsync(&counters->next, 0, sizeof(unsigned long long), st));
    run.walk_level(lo, hi, q0, op);
    drain_kernel<<<g->sm_count * 2, kThreads, 0, st>>>(op, q1, counters);
    ++stats.kernel_launches;
    if ((rc = run.read())) return rc;
    lo = hi;
    hi += run.host.next;
  }
  stats.trimmed = run.host.listed + run.host.trimmed;
  uint64_t live = n - stats.trimmed;

  // forward-backward from the pivot
  if (live > 0) {
    MGB_CUDA(cub::DeviceReduce::ArgMax(cub_tmp, argmax_bytes, keys, pivot_key, pivot, static_cast<int64_t>(n), st));
    seed_kernel<<<1, 1, 0, st>>>(pivot, 1, mark, q0, counters);
    ++stats.kernel_launches;
    uint64_t reached = 0;
    if ((rc = run.frontier(ForwardOp{{}, out, rep, mark, nullptr, nullptr, 0}, 0, 1, &reached))) return rc;
    seed_kernel<<<1, 1, 0, st>>>(pivot, 2, mark, q0, counters);
    ++stats.kernel_launches;
    if ((rc = run.frontier(BackwardOp{{}, in, mark, &counters->pivot_rep, nullptr, nullptr, 0}, 0, 1, &reached)))
      return rc;
    pivot_component_kernel<<<grid, kThreads, 0, st>>>(n, mark, rep, counters);
    ++stats.kernel_launches;
    if ((rc = run.read())) return rc;
    stats.pivot_component = run.host.pivot_size;
    live -= stats.pivot_component;
  }

  // colouring rounds until no vertex is live
  while (live > 0) {
    if ((rc = run.poll())) return rc;
    ++stats.coloring_rounds;
    MGB_CUDA(cudaMemsetAsync(&counters->next, 0, sizeof(unsigned long long), st));
    colour_init_kernel<<<grid, kThreads, 0, st>>>(n, rep, colour, q0, counters);
    ++stats.kernel_launches;
    uint64_t reached = 0;
    if ((rc = run.frontier(PropagateOp{{}, out, rep, colour, snap, queued, nullptr, nullptr, 0}, 0, live, &reached)))
      return rc;
    MGB_CUDA(cudaMemsetAsync(&counters->listed, 0, sizeof(unsigned long long), st));
    roots_kernel<<<grid, kThreads, 0, st>>>(n, colour, rep, q0, counters);
    ++stats.kernel_launches;
    if ((rc = run.read())) return rc;
    const uint64_t roots = run.host.listed;
    if ((rc = run.frontier(CollectOp{{}, in, colour, rep, nullptr, nullptr, 0}, 0, roots, &reached))) return rc;
    if (roots + reached > live) {
      set_error("strongly connected components: more vertices collected than were live (internal error)");
      return MGB200_ERR_CUDA;
    }
    live -= roots + reached;
  }

  // sizes, then the numbering
  size_kernel<<<grid, kThreads, 0, st>>>(n, rep, size);
  ++stats.kernel_launches;
  MGB_CUDA(cub::DeviceReduce::Max(cub_tmp, max_bytes, size, largest, n, st));
  MGB_CUDA(number_sets(n, rep, scan, component, cub_tmp, &number_bytes, grid, st));
  ++stats.kernel_launches;
  MGB_CUDA(cudaGetLastError());
  MGB_CUDA(cudaEventRecord(g->ev1, st));

  uint32_t tail[2] = {0, 0}, largest_host = 0;  // scan[n - 1], rep[n - 1]
  MGB_CUDA(cudaMemcpyAsync(&tail[0], scan + n - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaMemcpyAsync(&tail[1], rep + n - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaMemcpyAsync(&largest_host, largest, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  if ((rc = run.fetch())) return rc;
  float ms = 0.f;
  MGB_CUDA(cudaEventElapsedTime(&ms, g->ev0, g->ev1));
  MGB_CUDA(cudaMemcpyAsync(component_out, component, n * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  stats.components = static_cast<uint64_t>(tail[0]) + (tail[1] == n - 1 ? 1 : 0);
  stats.largest_component = largest_host;
  stats.edges_inspected = run.host.inspected;
  stats.run_ms = ms;
  if (stats_out) *stats_out = stats;
  return MGB200_OK;
}

int mgb200_strongly_connected_components(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                         int64_t *component_out) {
  if (n > 0 && !component_out) {
    set_error("strongly connected components: component_out is null");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  mgb200_bfs_graph *g = nullptr;
  int rc = mgb200_bfs_graph_create_host(0, n, m, from, to, &g);
  if (rc) return rc;
  rc = mgb200_scc_run(g, nullptr, nullptr, component_out, nullptr);
  mgb200_bfs_graph_destroy(g);
  return rc;
}

}  // extern "C"

// memgraph_b200/csrc/pagerank_kernels.cu -- the power iteration as hand-written sm_90a kernels.
//
// What is computed (reference: mage/cpp/pagerank_module/algorithm/pagerank.cpp):
//   r_{k+1}[v] = (1-d)/N + d * sum_{(u->v) in E} r_k[u] / outdeg(u)          :86-96, :104-112, :221-226
//   continue iff k+1 != max_iterations and max_v |r_{k+1}[v] - r_k[v]| > eps  :138-150
//   result = r_K / sum(r_K)                                                   :156-161
// The reference pushes along source-ordered edges into per-thread N-vectors; here the same sum is
// PULLED per destination row from contrib[u] = r_k[u]/outdeg(u), which is computed once per vertex
// with an IEEE division (bit-identical to the reference's per-edge quotient).  Only the order of
// the additions inside a row differs from the reference (ascending source label here).
//
// Roofline: HBM-bound sparse gather, no tensor cores.  Algorithmic bytes per iteration
// 12*E + 24*N (SURVEY 8d).  Per edge: one coalesced 4-byte index read (streamed, evict-first) and
// one 8-byte gather of contrib[]; per row: rank RMW in place, out-degree read, contrib write.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "core.hpp"

namespace mgb200 {
namespace {

constexpr int kBlockThreads = 256;
constexpr int kWarpsPerBlock = kBlockThreads / 32;
constexpr unsigned kFull = 0xffffffffu;
#ifndef MGB_UNROLL
#define MGB_UNROLL 8   // heavy-row segments: gathers in flight per lane
#endif
constexpr int kUnroll = MGB_UNROLL;

// ---- small PTX helpers ---------------------------------------------------------------------------

// Streaming read of an index word: read once per iteration, keep it out of the way of the
// gathered vector in L1/L2 (ld.global.nc, no L1 allocation, L2 evict-first policy).
__device__ __forceinline__ uint64_t make_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
#ifndef MGB_IDX_HINT
#define MGB_IDX_HINT 1     // 1: index stream no L1 allocation + L2 evict_first, 0: plain read-only loads
#endif
#ifndef MGB_EPI_HINT
#define MGB_EPI_HINT 1     // 1: rank / out-degree / contrib_out traffic evict_first, 0: default policy
#endif
#ifndef MGB_GATHER_POLICY
#define MGB_GATHER_POLICY 1  // 0: plain ld.global.nc, 1: range(evict_last hot prefix, evict_first tail), 2: all evict_last
#endif
__device__ __forceinline__ uint32_t ld_index(const uint32_t *p, uint64_t pol) {
#if MGB_IDX_HINT
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
#else
  (void)pol;
  return __ldg(p);
#endif
}
// Gather of one contribution: read-only path; reuse across CTAs lives in L2.
__device__ __forceinline__ double ld_contrib(const double *p, uint64_t pol) {
#if MGB_GATHER_POLICY
  double v;
  asm volatile("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
  return v;
#else
  (void)pol;
  return __ldg(p);
#endif
}
// L2 / L1 residency plan (microbenchmarks: scripts/l2_bench.cu, scripts/gather_bench.cu): random gathers are several
// times faster while the gathered set fits the part of L2 that holds it than from HBM; an SM issues one L2 request per
// cycle, so every L1 hit is a request saved, and with plain LRU the gathers that miss evict the hottest lines.  Labels
// are sorted by degree, so "hot" is a property of the label alone:
//   one partition : the hot vertices are the PREFIX of contrib[]            -> local index = label
//   P partitions  : sorted positions are dealt round-robin, every partition's label range starts with ITS
//                   hottest vertices                                          -> local index = label - start[owner]
// local < l2_hot: L2 evict_last, else evict_first (like every other stream: indices, rank, out-degree, contrib_out);
// local < l1_hot: may allocate in L1 (evict_last), else bypasses it.
struct GatherWindow {
  uint32_t hot_bytes;    // single partition: primary (evict_last) span of the range policy, from contrib_in
  uint32_t total_bytes;  // whole vector (secondary span: evict_first)
  uint32_t l1_hot;       // local indices below this may allocate in L1
  uint32_t l2_hot;       // local indices below this are L2 evict_last (multi-partition form)
  uint32_t world;        // number of partitions
  uint32_t table_n;      // labels held in the shared-memory hot table (0 = none); P partitions: table_n / P per owner
  uint32_t path;         // kernel instantiation: kPathRange / kPathLookup / kPathFlags (below)
  uint32_t start[kMaxPeers];  // first global label of every partition
};
constexpr uint32_t kL1Plain = kNoL1Hints;  // GatherWindow::l1_hot value meaning "no L1 hints"
// How a gather learns whether its source is hot:
//   kPathRange  one partition: a createpolicy.range over the prefix decides L2, `label < l1_hot` decides L1;
//   kPathLookup P partitions, plain indices: owner found by <= 7 compare/selects per gather, kept for graphs with
//               >= 2^30 vertices and as the A/B baseline;
//   kPathFlags  the hotness was computed ONCE at build time and rides in bits 31/30 of the stored index
//               (graph_build.cu IndexFlags): two bit tests per gather, no per-partition table in the kernel.
constexpr int kPathRange = 0, kPathLookup = 1, kPathFlags = 2;
struct GatherPolicy {
  uint64_t hot;   // single partition: the range policy; else fractional evict_last
  uint64_t cold;  // fractional evict_first
};
__device__ __forceinline__ GatherPolicy make_gather_policy(const double *contrib_in, const GatherWindow &w) {
  GatherPolicy p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p.cold));
  if (w.path == kPathRange && w.hot_bytes == 0) {  // MGB200_L2_HOT_MB=0: every gather evict_first, and no
    p.hot = p.cold;  // createpolicy.range with a zero primary size (a case the PTX ISA does not describe)
  } else if (w.path == kPathRange) {  // single partition, or partition-unaware legacy mode: one range policy over the prefix
    asm volatile("createpolicy.range.global.L2::evict_last.L2::evict_first.b64 %0, [%1], %2, %3;"
                 : "=l"(p.hot)
                 : "l"(contrib_in), "r"(w.hot_bytes), "r"(w.total_bytes));
  } else {
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p.hot));
  }
  return p;
}
// The hottest labels live in shared memory (kTable): an L2 request is what the SMs run out of (one per SM per clock),
// and the degree-sorted labelling makes "hottest" a prefix -- 21 % of all gathers of RMAT-26 go to the first 16 K
// labels, 27 % to the first 28 K (scripts/topk_share.py).  One partition: slot = label (label < table_n).  Several
// partitions: the build stored the slot in the index itself, code 01 in bits 31/30 (graph_build.cu IndexFlags).
// kStaged (the SELL walk on the range path): an index with kIdxStaged set is a slot of `staged` (graph_build.cu sell_staging),
// filled by the block pass of its source's block; it is read once per gather, evict-first in L2.
#ifndef MGB_STAGE_L1
#define MGB_STAGE_L1 1  // staged reads: 1 default L1 allocation (neighbouring columns share sectors), 0 no_allocate
#endif
template <int kPath, bool kSelectL2 = true, bool kTable = false, bool kStaged = false>
__device__ __forceinline__ double ld_contrib_at(const double *base, uint32_t src, const GatherPolicy &gp,
                                                const GatherWindow &w, const double *table = nullptr,
                                                const double *staged = nullptr) {
  if (kTable) {
    if (kPath == kPathFlags) {
      if ((src >> 30) == 1u) return table[src & kIdxLabelMask];
    } else if (src < w.table_n) {
      return table[src];
    }
  }
  if (kStaged && kPath == kPathRange && (src & kIdxStaged)) {
    const double *p = staged + (src & ~kIdxStaged);
    double v;
#if MGB_STAGE_L1
    asm volatile("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(gp.cold));
#else
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(gp.cold));
#endif
    return v;
  }
  uint32_t label = src;
  uint64_t pol = gp.hot;
  bool l1_hot;
  if (kPath == kPathFlags) {
    label = src & kIdxLabelMask;
    if (kSelectL2) pol = (src & kIdxL2Hot) ? gp.hot : gp.cold;  // else: every gather of this kernel evict_last
    l1_hot = (src & kIdxL1Hot) != 0;
  } else if (kPath == kPathLookup) {
    uint32_t s0 = 0;
#pragma unroll
    for (int q = 1; q < kMaxPeers; ++q)
      if (q < static_cast<int>(w.world) && src >= w.start[q]) s0 = w.start[q];
    const uint32_t local = src - s0;
    pol = local < w.l2_hot ? gp.hot : gp.cold;
    l1_hot = local < w.l1_hot;
  } else {
    l1_hot = src < w.l1_hot;
  }
  const double *p = base + label;
  double v;
  if (w.l1_hot == kL1Plain) {  // default L1 policy for every gather
    asm volatile("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
  } else if (l1_hot) {
    asm volatile("ld.global.nc.L1::evict_last.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
  } else {
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
  }
  return v;
}
__device__ __forceinline__ double ld_stream_f64(const double *p, uint64_t pol) {
#if MGB_EPI_HINT
  double v;
  asm volatile("ld.global.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
  return v;
#else
  (void)pol;
  return *p;
#endif
}
__device__ __forceinline__ void st_stream_f64(double *p, double v, uint64_t pol) {
#if MGB_EPI_HINT
  asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(pol) : "memory");
#else
  (void)pol;
  *p = v;
#endif
}

__device__ __forceinline__ int ld_volatile_int(const int *p) { return *reinterpret_cast<const volatile int *>(p); }

__device__ __forceinline__ void st_release_sys_u64(unsigned long long *p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long *p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---- mbarrier / TMA bulk-copy helpers (hot table fill here, index ring in sell_stream.cuh) ---------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  }
}
// TMA bulk copy global -> shared (1-D, bytes multiple of 16), completion counted on the mbarrier.
__device__ __forceinline__ void tma_load_1d(uint32_t dst_smem, const void *src, uint32_t bytes, uint32_t bar,
                                            uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar), "l"(pol)
      : "memory");
}

// ---- per-row epilogue ------------------------------------------------------------------------------

struct RowEpilogue {
  double base;     // (1 - d) / N
  double damping;  // d
  double *rank;            // [local_rows]
  const uint32_t *outdeg;  // [n] by global label
  RowMap map;              // local row -> global label
  double *contrib_out[kMaxPeers];  // this iteration's output buffer on every partition (self included)
  int world;
  int self;                // this partition
  const uint8_t *need;     // [local_rows] bit q: partition q gathers this row's contribution; nullptr = everyone
  uint32_t store_mask;     // bit q: the epilogue stores into partition q's buffer (all ones; self only in the lone-partition profiling mode)
};

// max over the block of the rows' |delta| (callers start from -1.0 = "none seen"; NaN deltas never replace it, like
// the reference's `abs(...) > eps` is false for NaN) -> one atomicMax on bits + 1, so that 0 keeps meaning "none".
__device__ __forceinline__ void block_max_to_state(double local_max, IterState *state) {
  __shared__ double warp_max[kWarpsPerBlock];
  for (int o = 16; o > 0; o >>= 1) {
    const double other = __shfl_xor_sync(kFull, local_max, o);
    if (other > local_max) local_max = other;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) warp_max[warp] = local_max;
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = warp_max[0];
    for (int w = 1; w < kWarpsPerBlock; ++w)
      if (warp_max[w] > m) m = warp_max[w];
    if (m >= 0.0) atomicMax(&state->diff_bits, static_cast<unsigned long long>(__double_as_longlong(m)) + 1ull);
  }
}

// ---- init -------------------------------------------------------------------------------------------

// Zero in-degree rows never receive anything: their rank is (1-d)/N after the first iteration and stays
// there, and their contribution is (that rank)/outdeg.  Every partition knows every partition's zero-row
// label ranges (graph_build.cu), so all of it is set up locally -- no kernel in the iteration loop, no
// NVLink traffic: init writes rank = (1-d)/N for the own zero rows, contrib[0] = (1/N)/outdeg for every
// label and contrib[1] = ((1-d)/N)/outdeg for all zero-row labels; zero_refresh_kernel rewrites contrib[0]
// for the zero-row labels during iteration 1.  Their one-time delta |(1-d)/N - 1/N| enters iteration 0's
// L-infinity test through iter_end_kernel (extra_diff_bits).
struct ZeroRanges {
  uint64_t lo[kMaxPeers];
  uint64_t hi[kMaxPeers];
  int world;
};

// rank = 1/N (:199); contrib[0] = (1/N)/outdeg for EVERY label (each partition fills its own full
// copy, so iteration 0 needs no exchange); pad slots = 0.
__global__ void __launch_bounds__(kBlockThreads) init_kernel(uint64_t n, uint64_t local_rows, uint64_t local_nonzero,
                                                             double zero_rank, double *rank, const uint32_t *outdeg,
                                                             double *contrib0, double *contrib1, ZeroRanges zr,
                                                             IterState *state) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const double r0 = 1.0 / static_cast<double>(n);
  for (uint64_t i = tid; i < n; i += stride) {
    const uint32_t od = outdeg[i];
    if (od) contrib0[i] = __ddiv_rn(r0, static_cast<double>(od));
  }
  for (int q = 0; q < kMaxPeers; ++q) {
    if (q >= zr.world) break;
    for (uint64_t i = zr.lo[q] + tid; i < zr.hi[q]; i += stride) {
      const uint32_t od = outdeg[i];
      if (od) contrib1[i] = __ddiv_rn(zero_rank, static_cast<double>(od));
    }
  }
  for (uint64_t i = tid; i < local_rows; i += stride) rank[i] = i < local_nonzero ? r0 : zero_rank;
  if (tid == 0) {
    contrib0[n] = 0.0;
    contrib1[n] = 0.0;
    state->diff_bits = 0ull;
    state->iterations = 0ull;
    state->last_diff = 0.0;
    state->local_sum = 0.0;
    state->rank_sum = 0.0;
    state->done = 0;
    state->error = 0;
    state->abort_req = 0;
    state->aborted = 0;
  }
}

// iteration 1 only: contrib[0] of the zero-row labels moves from (1/N)/outdeg to ((1-d)/N)/outdeg
__global__ void __launch_bounds__(kBlockThreads) zero_refresh_kernel(double zero_rank, const uint32_t *outdeg,
                                                                     double *contrib0, ZeroRanges zr,
                                                                     IterState *state) {
  if (ld_volatile_int(&state->done)) return;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t pol = make_evict_first_policy();
  for (int q = 0; q < kMaxPeers; ++q) {
    if (q >= zr.world) break;
    for (uint64_t i = zr.lo[q] + tid; i < zr.hi[q]; i += stride) {
      const uint32_t od = ld_index(outdeg + i, pol);
      if (od) st_stream_f64(contrib0 + i, __ddiv_rn(zero_rank, static_cast<double>(od)), pol);
    }
  }
}

// ---- SELL-32 rows: one lane per row, coalesced column-major index reads -----------------------------

// Row epilogue as a separate, perfectly coalesced elementwise pass over rows [first_row, end_row) whose gathered sums
// lie in sums[r - first_row]; used for the SELL class (its own kernel on the side stream) and for the heavy rows
// (after heavy_rowsum_kernel).  Fused into the gather kernels, the rank and out-degree loads, the FP64 division and
// the stores sit at the end of every slice's dependency chain and drain the warp's memory pipeline once per ~24
// columns.  This pass takes kEpiRows rows per trip and issues every load of the trip before the first use, as plain
// streaming loads (ld/st.global.cs) the compiler may hoist, instead of two dependent DRAM round trips per row.
//
//   rank_next = base + d * acc as two separately rounded operations, like the reference's
//   `rank_next[i] += damping_factor * block[i]` compiled without FMA contraction (:109-111);
//   contribution = rank_next / outdeg with an IEEE division (:93), once per vertex instead of once per edge.
constexpr int kEpiRows = 4;
__global__ void __launch_bounds__(kBlockThreads) row_epilogue_kernel(uint64_t first_row, uint64_t end_row,
                                                                     const double *sums, IterState *state,
                                                                     const RowEpilogue ep) {
  if (ld_volatile_int(&state->done)) return;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  double local_max = -1.0;
  for (uint64_t r0 = first_row + static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r0 < end_row;
       r0 += stride * kEpiRows) {
    double acc[kEpiRows], prev[kEpiRows];
    uint32_t od[kEpiRows], need[kEpiRows];
    uint64_t label[kEpiRows];
#pragma unroll
    for (int j = 0; j < kEpiRows; ++j) {
      const uint64_t r = r0 + j * stride;
      const bool ok = r < end_row;
      label[j] = ep.map.label_of_local(ok ? r : first_row);
      acc[j] = ok ? __ldcs(sums + (r - first_row)) : 0.0;
      prev[j] = ok ? __ldcs(ep.rank + r) : 0.0;
      od[j] = ok ? __ldcs(ep.outdeg + label[j]) : 0u;
      // push only to the partitions that have an in-edge from this vertex (graph_build.cu need_mask_kernel)
      need[j] = (ok && ep.need) ? (static_cast<uint32_t>(__ldcs(ep.need + r)) | (1u << ep.self)) : 0xFFu;
    }
#pragma unroll
    for (int j = 0; j < kEpiRows; ++j) {
      const uint64_t r = r0 + j * stride;
      if (r < end_row) {
        const double next = __dadd_rn(ep.base, __dmul_rn(ep.damping, acc[j]));
        __stcs(ep.rank + r, next);
        // A vertex without out-edges is never a gather source, so its contribution is never read: no division, no
        // store, and -- what matters across GPUs -- no NVLink push.  Labels are sorted by (in-degree, out-degree)
        // descending, so these vertices are the contiguous tail of every in-degree class: whole warps skip.
        if (od[j] != 0) {
          const double c = __ddiv_rn(next, static_cast<double>(od[j]));
          const uint32_t to = need[j] & ep.store_mask;
#pragma unroll
          for (int q = 0; q < kMaxPeers; ++q)
            if (q < ep.world && ((to >> q) & 1u)) __stcs(ep.contrib_out[q] + label[j], c);  // q != self: NVLink store
        }
        const double d = fabs(next - prev[j]);
        if (d > local_max) local_max = d;  // NaN never replaces it, like the reference's `abs(...) > eps`
      }
    }
  }
  block_max_to_state(local_max, state);
}

struct SellArgs {
  const uint64_t *colbase;
  const uint32_t *idx;
  const double *w;       // edge weights parallel to idx (weighted variants only, else nullptr)
  const WorkItem *work;  // [n_work] contiguous slice runs of ~equal cost, descending width (graph_build.cu)
  uint32_t n_work;
  WorkQueue *queue;      // ticket counter of this launch (rewound by the last CTA to leave)
  uint32_t mode;         // 0 tickets in list order (default), 1 static round-robin (A/B baseline)
  uint64_t first_row;    // local row of slice 0, lane 0
  uint64_t end_row;      // first local row past the SELL class
  const double *contrib_in;
  GatherWindow window;
  IterState *state;
  double *sums;  // [n_sell] per-row sums of gathered contributions (consumed by row_epilogue_kernel)
  const double *stage_val;  // staged values of the entries marked kIdxStaged (filled by the block passes), or nullptr
};

// Tunables (compile-time; variants: scripts/build_variants.py)
#ifndef MGB_SELL_UNROLL
#define MGB_SELL_UNROLL 8      // columns per batch (gathers in flight per lane)
#endif
#ifndef MGB_SELL_MIN_BLOCKS
#define MGB_SELL_MIN_BLOCKS 3  // resident CTAs/SM requested from ptxas (register cap = 65536 / (256 * this)): at 4 the
                               // walk is capped at 64 registers and spills 152 bytes; at 3 it takes 80 and spills
                               // none, 6 % less SELL time despite 24 instead of 32 warps per SM (DESIGN.md §4)
#endif
constexpr int kSellUnroll = MGB_SELL_UNROLL;

// SELL-32 rows: one lane per row, a warp walks a WORK ITEM = a contiguous run of slices, i.e. one contiguous span of
// sell_idx, as ONE stream of columns: index batch k+1 is requested before the gathers of batch k are consumed, across
// slice boundaries -- a boundary only decides where the running sum is stored.  (The first version restarted its
// pipeline at every slice: an exposed round trip per slice, 22 per warp on a 1/8 partition, and every run of narrow
// slices degenerated to `width` gathers in flight.)  Items have about equal cost and are handed out in descending-width
// order through a ticket counter, so a warp that drew cheap work (or sits on an SM with the longer way to L2) simply takes
// more; the queue is software-pipelined (record of item i+1 and ticket of item i+2 in flight while item i is gathered).
// mode 1 deals the items round-robin instead (no atomics) -- the A/B baseline of the ticket queue.
template <int kPath, bool kTable, bool kWeighted = false>
__device__ __forceinline__ void sell_walk(const SellArgs &a, const double *table) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = static_cast<int>(blockDim.x >> 5);
  const uint64_t pol = make_evict_first_policy();
  const GatherPolicy gpol = make_gather_policy(a.contrib_in, a.window);
  unsigned long long static_next = static_cast<unsigned long long>(blockIdx.x) * warps_per_block + (threadIdx.x >> 5);
  const unsigned long long warps_total = static_cast<unsigned long long>(gridDim.x) * warps_per_block;
  auto draw = [&]() -> unsigned long long {
    if (a.mode == 1) {
      const unsigned long long t = static_next;
      static_next += warps_total;
      return t;
    }
    return lane == 0 ? atomicAdd(&a.queue->ticket, 1ull) : 0ull;
  };
  // lanes 0..3 fetch the four words of an item record (one 32-byte sector)
  auto fetch = [&](uint32_t t) -> uint64_t {
    return (lane < 4 && t < a.n_work) ? reinterpret_cast<const uint64_t *>(a.work + t)[lane] : 0ull;
  };
  uint32_t t_cur = static_cast<uint32_t>(min(__shfl_sync(kFull, draw(), 0), static_cast<unsigned long long>(a.n_work)));
  unsigned long long pending = draw();  // ticket of the item after the first
  uint64_t rec = fetch(t_cur);
  while (t_cur < a.n_work) {
    const uint64_t s_begin = __shfl_sync(kFull, rec, 0), s_end = __shfl_sync(kFull, rec, 1);
    const uint64_t col_begin = __shfl_sync(kFull, rec, 2), col_end = __shfl_sync(kFull, rec, 3);
    // next item: its ticket was drawn one item ago; request its record now, and draw the ticket after it
    t_cur = static_cast<uint32_t>(min(__shfl_sync(kFull, pending, 0), static_cast<unsigned long long>(a.n_work)));
    rec = fetch(t_cur);
    pending = draw();
    if (s_begin >= s_end) continue;
    // slice ends: lane l holds colbase[block + l + 1] for a block of 32 slices (one coalesced load per 32 slices)
    uint64_t s = s_begin, s_block = s_begin;
    uint64_t ends = (s_block + lane + 1 <= s_end) ? a.colbase[s_block + lane + 1] : col_end;
    uint64_t slice_end = __shfl_sync(kFull, ends, 0);
    const uint32_t *p = a.idx + col_begin * kSliceRows + lane;  // column c of the span: p[(c - col_begin) * 32]
    const uint64_t ncols = col_end - col_begin;
    double acc = 0.0;
    uint32_t nxt[kSellUnroll];
#pragma unroll
    for (int j = 0; j < kSellUnroll; ++j)
      if (static_cast<uint64_t>(j) < ncols) nxt[j] = ld_index(p + static_cast<size_t>(j) * kSliceRows, pol);
    for (uint64_t k = 0; k < ncols; k += kSellUnroll) {
      uint32_t src[kSellUnroll];
      double v[kSellUnroll];
#pragma unroll
      for (int j = 0; j < kSellUnroll; ++j) src[j] = nxt[j];
#ifdef MGB_SELL_HOT_ONLY_FROM  // bound measurement only (wrong ranks): sources >= this label read the zero slot n
      if (kPath == kPathRange) {
#pragma unroll
        for (int j = 0; j < kSellUnroll; ++j)
          if (src[j] >= MGB_SELL_HOT_ONLY_FROM) src[j] = a.window.total_bytes / sizeof(double) - 1;
      }
#endif
#pragma unroll
      for (int j = 0; j < kSellUnroll; ++j)  // the next batch of indices travels while this batch is gathered
        if (k + kSellUnroll + j < ncols) nxt[j] = ld_index(p + static_cast<size_t>(k + kSellUnroll + j) * kSliceRows, pol);
      double wv[kSellUnroll];
      if (kWeighted) {
        const double *pw = a.w + col_begin * kSliceRows + lane;
#pragma unroll
        for (int j = 0; j < kSellUnroll; ++j)
          if (k + j < ncols) wv[j] = ld_stream_f64(pw + static_cast<size_t>(k + j) * kSliceRows, pol);
      }
#pragma unroll
      for (int j = 0; j < kSellUnroll; ++j)
        if (k + j < ncols)
          v[j] = ld_contrib_at<kPath, true, kTable, !kWeighted>(a.contrib_in, src[j], gpol, a.window, table, a.stage_val);
      if (kWeighted) {
#pragma unroll
        for (int j = 0; j < kSellUnroll; ++j)
          if (k + j < ncols) v[j] = __dmul_rn(wv[j], v[j]);
      }
#pragma unroll
      for (int j = 0; j < kSellUnroll; ++j) {
        if (k + j < ncols) {
          acc += v[j];  // fixed order inside a row: ascending source label
          const uint64_t col_next = col_begin + k + j + 1;
          while (col_next == slice_end && s < s_end) {  // (a zero-width slice would store 0 for its rows right here)
            const uint64_t row = a.first_row + s * kSliceRows + lane;
            if (row < a.end_row) a.sums[row - a.first_row] = acc;  // epilogue runs as its own elementwise kernel
            acc = 0.0;
            ++s;
            if (s < s_end) {
              if (s - s_block == 32) {
                s_block = s;
                ends = (s_block + lane + 1 <= s_end) ? a.colbase[s_block + lane + 1] : col_end;
              }
              slice_end = __shfl_sync(kFull, ends, static_cast<int>(s - s_block));
            }
          }
        }
      }
    }
  }
  if (a.mode == 1) return;
  // the last CTA to leave rewinds the queue for the next launch (every ticket of this launch has been drawn by then)
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int left = atomicAdd(&a.queue->ctas_done, 1u);
    if (left == gridDim.x - 1) {
      a.queue->ticket = 0ull;
      a.queue->ctas_done = 0u;
      __threadfence();
    }
  }
}


template <int kPath>
__global__ void __launch_bounds__(kBlockThreads, MGB_SELL_MIN_BLOCKS) sell_rows_kernel(const SellArgs a) {
  if (ld_volatile_int(&a.state->done)) return;
  sell_walk<kPath, false>(a, nullptr);
}

// every gathered value multiplied by its edge weight (cuGraph-semantics variants, one partition)
__global__ void __launch_bounds__(kBlockThreads, MGB_SELL_MIN_BLOCKS) sell_rows_weighted_kernel(const SellArgs a) {
  if (ld_volatile_int(&a.state->done)) return;
  sell_walk<kPathRange, false, true>(a, nullptr);
}

// The same walk with the hot table: ONE CTA per SM so that the SM holds one copy of the table; filled once per launch --
// one partition: TMA bulk copies (cp.async.bulk, 32 KiB each, completion on an mbarrier, L2 evict-last) of the
// contiguous label prefix; several partitions: one window per owner, whose first label is only 8-byte aligned, so the
// threads load it cooperatively.  768 threads = the plain kernel's 24 warps per SM, with up to 85 registers each: at
// 1024 threads ptxas caps the walk at 64 registers and it spills, as the plain walk did at 4 CTAs per SM (DESIGN.md §4).
#ifndef MGB_TABLE_THREADS
#define MGB_TABLE_THREADS 768
#endif
constexpr int kTableThreads = MGB_TABLE_THREADS;
template <int kPath>
__global__ void __launch_bounds__(kTableThreads, 1) sell_rows_table_kernel(const SellArgs a) {
  extern __shared__ __align__(128) unsigned char table_smem[];
  __shared__ __align__(8) unsigned long long fill_bar;
  if (ld_volatile_int(&a.state->done)) return;
  double *table = reinterpret_cast<double *>(table_smem);
  const uint32_t table_n = a.window.table_n;
  if (kPath == kPathFlags) {
    const uint32_t per = table_n / a.window.world;
    for (uint32_t q = 0; q < a.window.world; ++q)
      for (uint32_t i = threadIdx.x; i < per; i += blockDim.x)
        table[q * per + i] = __ldg(a.contrib_in + a.window.start[q] + i);
    __syncthreads();
  } else {
    const uint32_t bar = smem_u32(&fill_bar);
    if (threadIdx.x == 0) {
      mbar_init(bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      uint64_t keep;
      asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(keep));
      const uint32_t bytes = table_n * static_cast<uint32_t>(sizeof(double));
      mbar_expect_tx(bar, bytes);
      for (uint32_t off = 0; off < bytes; off += 32768u)
        tma_load_1d(smem_u32(table_smem + off), reinterpret_cast<const unsigned char *>(a.contrib_in) + off,
                    min(32768u, bytes - off), bar, keep);
    }
    __syncthreads();  // the barrier is initialised before anyone waits on it
    mbar_wait(bar, 0);
  }
  sell_walk<kPath, true>(a, table);
}

#include "sell_stream.cuh"

// ---- heavy rows: one warp per fixed-size edge segment, then one warp per row ------------------------

// Tile chunks (graph_build.cu 7c): a CTA copies one tile of contrib into shared memory with TMA bulk copies and serves
// every chunk of that tile from it -- per edge a 2-byte offset and a shared-memory read instead of a 4-byte index and
// an L2 request.  Slices are tile-major and cut into RUNS of about equal cost, several per SM; one persistent CTA per SM
// draws runs from a ticket in tile order, so a CTA that drew cheap runs simply takes more, and its next run lies in the
// tile it holds or in a later one (it refills only when the tile changes).  Inside a run the CTA's warps draw GROUPS of
// consecutive slices from a shared counter and walk each group as one stream of columns (tile_walk).
struct TileArgs {
  const uint16_t *idx;          // [32 * columns] tile offsets, column-major per slice
  const uint64_t *colbase;      // [slices + 1]
  const uint32_t *slice_tile;   // [slices]
  const uint64_t *slot;         // [32 * slices] partial of each lane's chunk, ~0 = padding lane
  const uint64_t *tile_slice_first;  // [tiles + 1]
  const uint32_t *tile_base, *tile_load;  // [tiles] first label (even) and labels copied (even)
  const uint64_t *work_begin;   // [n_work + 1] first slice of every run
  uint32_t n_work;
  WorkQueue *queue;             // ticket of the runs (rewound by the last CTA to leave)
  uint32_t tile_labels;         // T: shared slot T holds the 0.0 every padding offset reads
  const double *contrib_in;
  double *seg_partial;
  IterState *state;
};
constexpr int kTileThreads = 512;
constexpr int kTileWarps = kTileThreads / 32;
constexpr int kTileUnroll = 16;
constexpr int kTileGroupMax = 31;     // slices per group: its column bases, both ends included, fill one warp-wide load
constexpr int kTileGroupsPerWarp = 4; // groups a warp draws from a run's part of one tile, on average
constexpr int kTileEpiCtas = 2;  // CTAs per SM of the side-stream SELL epilogue next to heavy_tiles_kernel
__device__ __forceinline__ uint16_t ld_index16(const uint16_t *p, uint64_t pol) {
  uint16_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u16 %0, [%1], %2;" : "=h"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ uint64_t ld_slot(const uint64_t *p, uint64_t pol) {
  uint64_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
  return v;
}

// One warp's share of slices [.., run_end) of the loaded tile.  A ticket on `next_slice` hands out a group of `group`
// consecutive slices, which is one contiguous span of tile_idx because colbase is monotone; the warp walks the span as
// ONE stream of columns (offset batch k+1 travels while batch k is summed), and a slice boundary only decides where the
// lane's sum is stored -- narrow slices cost columns, not round trips.  The next group's ticket and column bases travel
// while the current group is summed, and a slice's partial slots are requested two slices ahead.  A lane still adds its
// chunk alone, from 0.0, in ascending source order: the partials are the bits a slice-by-slice walk gives.
__device__ __forceinline__ void tile_walk(const TileArgs &a, const double *tile, unsigned long long *next_slice,
                                          uint64_t run_end, uint32_t group, int lane, uint64_t pol) {
  auto draw = [&]() -> uint64_t {
    unsigned long long t = 0;
    if (lane == 0) t = atomicAdd(next_slice, static_cast<unsigned long long>(group));
    return __shfl_sync(kFull, t, 0);
  };
  // lane l: colbase[first + l], up to the end of the group's last slice
  auto bases = [&](uint64_t first) -> uint64_t {
    return (first < run_end && first + lane <= min(first + group, run_end)) ? a.colbase[first + lane] : 0ull;
  };
  auto slot_of = [&](uint64_t s, uint64_t end) -> uint64_t {
    return s < end ? ld_slot(a.slot + s * kSliceRows + lane, pol) : ~0ull;
  };
  uint64_t my = draw();
  uint64_t base = bases(my);
  while (my < run_end) {
    const uint64_t my_next = draw();
    const uint64_t base_next = bases(my_next);
    const uint64_t my_end = min(my + group, run_end);
    const uint64_t c0 = __shfl_sync(kFull, base, 0);
    const uint32_t ncols = static_cast<uint32_t>(__shfl_sync(kFull, base, static_cast<int>(my_end - my)) - c0);
    const uint32_t rel = static_cast<uint32_t>(base - c0);  // lane l: first column of slice my + l, from the group's start
    const uint16_t *p = a.idx + c0 * kSliceRows + lane;
    uint16_t nxt[kTileUnroll];
#pragma unroll
    for (int j = 0; j < kTileUnroll; ++j)
      if (static_cast<uint32_t>(j) < ncols) nxt[j] = ld_index16(p + static_cast<size_t>(j) * kSliceRows, pol);
    uint64_t s = my;
    uint64_t slot = slot_of(s, my_end), slot_ahead = slot_of(s + 1, my_end);
    uint32_t slice_end = __shfl_sync(kFull, rel, 1);
    double acc = 0.0;
    // column `col` (group-relative, one past the column just added) closes every slice that ends there
    auto close_slices = [&](uint32_t col) {
      while (col == slice_end) {  // every slice is >= 1 column wide (its longest chunk has an edge), so col >= 1 suffices
        if (slot != ~0ull) a.seg_partial[slot] = acc;
        acc = 0.0;
        ++s;
        slot = slot_ahead;
        slot_ahead = slot_of(s + 1, my_end);
        slice_end = s < my_end ? __shfl_sync(kFull, rel, static_cast<int>(s - my) + 1) : 0xFFFFFFFFu;
      }
    };
    for (uint32_t k = 0; k < ncols; k += kTileUnroll) {
      uint16_t off[kTileUnroll];
#pragma unroll
      for (int j = 0; j < kTileUnroll; ++j) off[j] = nxt[j];
#pragma unroll
      for (int j = 0; j < kTileUnroll; ++j)  // the next batch of offsets travels while this batch is summed
        if (k + kTileUnroll + j < ncols) nxt[j] = ld_index16(p + static_cast<size_t>(k + kTileUnroll + j) * kSliceRows, pol);
      if (k + kTileUnroll <= slice_end) {  // the whole batch lies inside the current slice
#pragma unroll
        for (int j = 0; j < kTileUnroll; ++j) acc += tile[off[j]];  // ascending source order inside the chunk
        close_slices(k + kTileUnroll);
      } else {
#pragma unroll
        for (int j = 0; j < kTileUnroll; ++j) {
          if (k + j < ncols) {
            acc += tile[off[j]];
            close_slices(k + j + 1);
          }
        }
      }
    }
    my = my_next;
    base = base_next;
  }
}

__global__ void __launch_bounds__(kTileThreads, 2) heavy_tiles_kernel(const TileArgs a) {  // <= 64 registers
  extern __shared__ __align__(128) unsigned char tile_smem[];
  __shared__ __align__(8) unsigned long long fill_bar;
  __shared__ unsigned long long next_slice;
  __shared__ uint32_t cta_run;
  // `done` is written by iter_end_kernel and, when a peer barrier times out, by barrier_kernel; both run on this
  // launch's stream, so every CTA of a launch reads the same value: either all of them draw tickets and count
  // themselves out below, or none touches the queue
  if (ld_volatile_int(&a.state->done)) return;
  const double *tile = reinterpret_cast<const double *>(tile_smem);
  const int lane = threadIdx.x & 31;
  const uint32_t bar = smem_u32(&fill_bar);
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    reinterpret_cast<double *>(tile_smem)[a.tile_labels] = 0.0;  // never overwritten: a fill copies <= T labels
  }
  const uint64_t pol = make_evict_first_policy();
  uint32_t phase = 0, cur_tile = 0xFFFFFFFFu;
  while (true) {
    if (threadIdx.x == 0)
      cta_run = static_cast<uint32_t>(min(atomicAdd(&a.queue->ticket, 1ull), static_cast<unsigned long long>(a.n_work)));
    __syncthreads();  // (first trip: the barrier is initialised before anyone waits on it)
    const uint32_t w = cta_run;
    if (w >= a.n_work) break;
    uint64_t s = a.work_begin[w];
    const uint64_t s_end = a.work_begin[w + 1];
    while (s < s_end) {
      const uint32_t t = a.slice_tile[s];
      const uint64_t run_end = min(s_end, a.tile_slice_first[t + 1]);
      if (threadIdx.x == 0) {
        next_slice = s;
        if (t != cur_tile) {
          // the previous tile's shared-memory reads (ordered by the __syncthreads below) precede the async-proxy writes
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          uint64_t keep;
          asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(keep));
          const uint32_t bytes = a.tile_load[t] * static_cast<uint32_t>(sizeof(double));
          const unsigned char *src = reinterpret_cast<const unsigned char *>(a.contrib_in + a.tile_base[t]);
          mbar_expect_tx(bar, bytes);
          for (uint32_t off = 0; off < bytes; off += 32768u)
            tma_load_1d(smem_u32(tile_smem + off), src + off, min(32768u, bytes - off), bar, keep);
        }
      }
      __syncthreads();
      if (t != cur_tile) {
        mbar_wait(bar, phase);
        phase ^= 1u;
        cur_tile = t;
      }
      // enough groups that the warps finish this part of the run together, few enough that a group is a long stream
      const uint32_t group = static_cast<uint32_t>(
          min(static_cast<uint64_t>(kTileGroupMax), max(uint64_t{1}, (run_end - s) / (kTileWarps * kTileGroupsPerWarp))));
      tile_walk(a, tile, &next_slice, run_end, group, lane, pol);
      __syncthreads();  // every warp is done with this part (and with next_slice) before the next fill
      s = run_end;
    }
    __syncthreads();  // every thread has read cta_run before the next ticket overwrites it (an empty run has no part)
  }
  // the last CTA to leave rewinds the ticket for the next launch (every run of this launch has been drawn by then)
  if (threadIdx.x == 0) {
    const unsigned int left = atomicAdd(&a.queue->ctas_done, 1u);
    if (left == gridDim.x - 1) {
      a.queue->ticket = 0ull;
      a.queue->ctas_done = 0u;
      __threadfence();
    }
  }
}

// Block passes (graph_build.cu block_slices): the heavy rows' in-edges from labels >= block_from, one label block per launch,
// so the block's part of contrib is read from HBM about once per pass instead of costing a sector per gather.  One warp
// per slice, one lane per chunk: the lane adds its chunk in ascending source order and stores the chunk's partial (no
// atomics, the same bits every run).
struct BlockArgs {
  const uint32_t *idx;      // [32 * columns] source labels, column-major per slice, pad = n
  const uint64_t *colbase;  // [slices + 1]
  const uint64_t *slot;     // [32 * slices] partial of each lane's chunk, ~0 = padding lane
  uint64_t slice_begin, slice_end;
  const double *block;      // contrib_in + first label of the block
  uint32_t block_bytes;      // evict_last span
  uint32_t tail_bytes;       // block .. the end of the vector (padding slot included): evict_first past the block
  const double *contrib_in;
  double *seg_partial;
  IterState *state;
  const uint32_t *stage_src;  // SELL entries staged from this block: stage_val[q] = contrib_in[stage_src[q]]
  double *stage_val;
  uint64_t stage_begin, stage_end;
};
constexpr int kStageUnroll = 4;  // staged copies per thread and trip: every label load issued before the first gather
__global__ void __launch_bounds__(kBlockThreads) cold_block_kernel(const BlockArgs a) {
  if (ld_volatile_int(&a.state->done)) return;
  const int lane = threadIdx.x & 31;
  const uint64_t warps_total = static_cast<uint64_t>(gridDim.x) * kWarpsPerBlock;
  const uint64_t pol = make_evict_first_policy();
  uint64_t gpol;  // evict_last over the block, evict_first past it (the padding slot); DESIGN.md §4: beats default priority
  asm volatile("createpolicy.range.global.L2::evict_last.L2::evict_first.b64 %0, [%1], %2, %3;"
               : "=l"(gpol)
               : "l"(a.block), "r"(a.block_bytes), "r"(a.tail_bytes));
  for (uint64_t s = a.slice_begin + static_cast<uint64_t>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5);
       s < a.slice_end; s += warps_total) {
    const uint64_t c0 = a.colbase[s], ncols = a.colbase[s + 1] - c0;
    const uint64_t slot = a.slot[s * kSliceRows + lane];
    const uint32_t *p = a.idx + c0 * kSliceRows + lane;
    double acc = 0.0;
    uint32_t nxt[kUnroll];
#pragma unroll
    for (int j = 0; j < kUnroll; ++j)
      if (static_cast<uint64_t>(j) < ncols) nxt[j] = ld_index(p + static_cast<size_t>(j) * kSliceRows, pol);
    for (uint64_t k = 0; k < ncols; k += kUnroll) {
      uint32_t src[kUnroll];
      double v[kUnroll];
#pragma unroll
      for (int j = 0; j < kUnroll; ++j) src[j] = nxt[j];
#pragma unroll
      for (int j = 0; j < kUnroll; ++j)  // the next batch of labels travels while this batch is gathered
        if (k + kUnroll + j < ncols) nxt[j] = ld_index(p + static_cast<size_t>(k + kUnroll + j) * kSliceRows, pol);
#pragma unroll
      for (int j = 0; j < kUnroll; ++j)
        if (k + j < ncols) v[j] = ld_contrib(a.contrib_in + src[j], gpol);
#pragma unroll
      for (int j = 0; j < kUnroll; ++j)
        if (k + j < ncols) acc += v[j];  // ascending source order inside the chunk
    }
    if (slot != ~0ull) a.seg_partial[slot] = acc;
  }
  // the SELL walk's values from this block (graph_build.cu sell_staging): edge-parallel, labels and stores streamed
  const uint64_t threads = static_cast<uint64_t>(gridDim.x) * kBlockThreads;
  for (uint64_t q0 = a.stage_begin + static_cast<uint64_t>(blockIdx.x) * kBlockThreads + threadIdx.x; q0 < a.stage_end;
       q0 += threads * kStageUnroll) {
    uint32_t src[kStageUnroll];
    double v[kStageUnroll];
#pragma unroll
    for (int j = 0; j < kStageUnroll; ++j)
      if (q0 + j * threads < a.stage_end) src[j] = ld_index(a.stage_src + q0 + j * threads, pol);
#pragma unroll
    for (int j = 0; j < kStageUnroll; ++j)
      if (q0 + j * threads < a.stage_end) v[j] = ld_contrib(a.contrib_in + src[j], gpol);
#pragma unroll
    for (int j = 0; j < kStageUnroll; ++j)
      if (q0 + j * threads < a.stage_end) st_stream_f64(a.stage_val + q0 + j * threads, v[j], pol);
  }
}

struct HeavyArgs {
  const uint64_t *heavy_ptr;
  const uint32_t *heavy_idx;
  const double *heavy_w;  // edge weights parallel to heavy_idx (weighted variants only)
  const uint32_t *seg_row;
  const uint64_t *seg_begin;
  const uint64_t *seg_slot;  // partial of each segment (nullptr: identity)
  const uint64_t *seg_first;
  double *seg_partial;
  double *row_sums;  // [n_heavy]
  uint64_t n_seg;
  uint64_t n_heavy;
  uint32_t segment_edges;
  const double *contrib_in;
  GatherWindow window;
  IterState *state;
};

#ifndef MGB_HEAVY_MIN_BLOCKS
#define MGB_HEAVY_MIN_BLOCKS 8  // 32 registers: occupancy beats the 8-16 B of spill (measured, r01_multi_gpu.md)
#endif
#ifndef MGB_HEAVY_PREFETCH
#define MGB_HEAVY_PREFETCH 0    // 1: request the next batch of segment indices before consuming the current gathers
#endif
#ifndef MGB_HEAVY_FLAGS_L2
#define MGB_HEAVY_FLAGS_L2 1    // flagged indices: 1 = per-load L2 hot/cold selection, 0 = L1 flag only
#endif
template <int kPath, bool kWeighted = false>
__global__ void __launch_bounds__(kBlockThreads, MGB_HEAVY_MIN_BLOCKS) heavy_segments_kernel(const HeavyArgs a) {
  constexpr bool kSelL2 = MGB_HEAVY_FLAGS_L2 != 0;
  if (ld_volatile_int(&a.state->done)) return;
  const int lane = threadIdx.x & 31;
  const uint64_t warps_total = static_cast<uint64_t>(gridDim.x) * kWarpsPerBlock;
  const uint64_t warp0 = static_cast<uint64_t>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5);
  const uint64_t pol = make_evict_first_policy();
  const GatherPolicy gpol = make_gather_policy(a.contrib_in, a.window);
  for (uint64_t g = warp0; g < a.n_seg; g += warps_total) {
    const uint32_t r = a.seg_row[g];
    const uint64_t e0 = a.seg_begin[g];
    const uint64_t row_end = a.heavy_ptr[r + 1];
    const uint64_t e1 = (e0 + a.segment_edges < row_end) ? e0 + a.segment_edges : row_end;
    double acc = 0.0;
    uint64_t e = e0 + lane;
#if MGB_HEAVY_PREFETCH
    // software pipeline like the SELL walk: the indices of batch k+1 are requested before the gathers of batch k are consumed
    uint32_t nxt[kUnroll];
    if (e + 32ull * (kUnroll - 1) < e1) {
#pragma unroll
      for (int j = 0; j < kUnroll; ++j) nxt[j] = ld_index(a.heavy_idx + e + 32ull * j, pol);
    }
#endif
    for (; e + 32ull * (kUnroll - 1) < e1; e += 32ull * kUnroll) {
      uint32_t src[kUnroll];
      double v[kUnroll];
#if MGB_HEAVY_PREFETCH
#pragma unroll
      for (int j = 0; j < kUnroll; ++j) src[j] = nxt[j];
      if (e + 32ull * kUnroll + 32ull * (kUnroll - 1) < e1) {
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) nxt[j] = ld_index(a.heavy_idx + e + 32ull * kUnroll + 32ull * j, pol);
      }
#else
#pragma unroll
      for (int j = 0; j < kUnroll; ++j) src[j] = ld_index(a.heavy_idx + e + 32ull * j, pol);
#endif
#pragma unroll
      for (int j = 0; j < kUnroll; ++j) v[j] = ld_contrib_at<kPath, kSelL2>(a.contrib_in, src[j], gpol, a.window);
      if (kWeighted) {
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) v[j] = __dmul_rn(ld_stream_f64(a.heavy_w + e + 32ull * j, pol), v[j]);
      }
#pragma unroll
      for (int j = 0; j < kUnroll; ++j) acc += v[j];
    }
    for (; e < e1; e += 32) {
      double v1 = ld_contrib_at<kPath, kSelL2>(a.contrib_in, ld_index(a.heavy_idx + e, pol), gpol, a.window);
      if (kWeighted) v1 = __dmul_rn(ld_stream_f64(a.heavy_w + e, pol), v1);
      acc += v1;
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(kFull, acc, o);  // fixed tree
    if (lane == 0) a.seg_partial[a.seg_slot ? a.seg_slot[g] : g] = acc;
  }
}

// per heavy row: segment partials summed in segment order (lane-strided, fixed shuffle tree) -> row_sums[r];
// the row epilogue then runs as row_epilogue_kernel over [0, n_heavy)
__global__ void __launch_bounds__(kBlockThreads) heavy_rowsum_kernel(const HeavyArgs a) {
  if (ld_volatile_int(&a.state->done)) return;
  const int lane = threadIdx.x & 31;
  const uint64_t warps_total = static_cast<uint64_t>(gridDim.x) * kWarpsPerBlock;
  const uint64_t warp0 = static_cast<uint64_t>(blockIdx.x) * kWarpsPerBlock + (threadIdx.x >> 5);
  for (uint64_t r = warp0; r < a.n_heavy; r += warps_total) {
    const uint64_t s0 = a.seg_first[r], s1 = a.seg_first[r + 1];
    double acc = 0.0;
    for (uint64_t s = s0 + lane; s < s1; s += 32) acc += a.seg_partial[s];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(kFull, acc, o);
    if (lane == 0) a.row_sums[r] = acc;
  }
}

// ---- cross-partition barrier over the flag pages (P == 1: degenerates to nothing) ---------------------

struct BarrierArgs {
  IterState *state;
  FlagPage *mine;
  FlagPage *peer[kMaxPeers];  // peer[q] = partition q's flag page as mapped on THIS device (self included)
  int rank, world;
  unsigned long long timeout_ns;
};

// One warp.  Publishes `payload_bits`/`payload_sum` into slot [rank] of every partition's flag page,
// then waits until every partition has arrived at the same sequence number.  All stores issued by
// earlier kernels of this stream (including remote contribution stores) are ordered before the
// release store by the kernel boundary plus the system-scope fence.
__device__ __forceinline__ bool warp_barrier_exchange(const BarrierArgs &b, unsigned long long seq,
                                                      unsigned long long payload_bits, double payload_sum) {
  const int lane = threadIdx.x & 31;
  const int par = static_cast<int>(seq & 1ull);
  bool ok = true;
  if (lane < b.world) {
    FlagPage *dst = b.peer[lane];
    st_relaxed_sys_u64(&dst->diff_bits[par][b.rank], payload_bits);
    st_relaxed_sys_u64(reinterpret_cast<unsigned long long *>(&dst->rank_sum[par][b.rank]),
                       static_cast<unsigned long long>(__double_as_longlong(payload_sum)));
    __threadfence_system();
    st_release_sys_u64(&dst->arrive[b.rank], seq);
    const unsigned long long t0 = global_timer_ns();
    while (ld_acquire_sys_u64(&b.mine->arrive[lane]) < seq) {
      if (global_timer_ns() - t0 > b.timeout_ns) {
        ok = false;
        break;
      }
      __nanosleep(64);
    }
  }
  return __all_sync(kFull, ok);
}

struct IterEndArgs {
  BarrierArgs bar;
  unsigned long long max_iterations;
  double eps;
  unsigned long long extra_diff_bits;  // iteration 0: the zero rows' |(1-d)/N - 1/N| (same on every partition)
};

// End of one iteration: all-reduce(max) of the L-infinity delta across partitions, then the
// reference's CheckContinueIterate (:138-150) evaluated identically on every partition.
__global__ void iter_end_kernel(const IterEndArgs a) {
  IterState *st = a.bar.state;
  if (ld_volatile_int(&st->done)) return;
  const int lane = threadIdx.x & 31;
  unsigned long long bits = st->diff_bits;  // bits(max delta) + 1, 0 = none
  if (a.extra_diff_bits > bits) bits = a.extra_diff_bits;
  // Abort is a COLLECTIVE decision: a partition whose host asked to stop publishes kAbortBits instead of its delta;
  // the max-reduce hands it to everyone, so all partitions leave the loop in the same iteration and their barrier
  // counters stay in step (a partition that returned on its own would leave the others waiting, then run ahead).
  if (ld_volatile_int(&st->abort_req)) bits = kAbortBits;
  bool ok = true;
  unsigned long long seq = st->barrier_seq;
  if (a.bar.world > 1) {
    seq += 1;
    ok = warp_barrier_exchange(a.bar, seq, bits, 0.0);
    unsigned long long other = 0ull;
    if (lane < a.bar.world) other = a.bar.mine->diff_bits[seq & 1ull][lane];
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long t = __shfl_xor_sync(kFull, other, o);
      if (t > other) other = t;
    }
    bits = other;
  }
  if (lane == 0) {
    st->barrier_seq = seq;
    const bool abort_all = bits == kAbortBits;
    const bool any_delta = bits != 0ull && !abort_all;
    const double diff = any_delta ? __longlong_as_double(static_cast<long long>(bits - 1ull)) : 0.0;
    st->iterations += 1ull;
    st->last_diff = diff;
    // :138-150 -- continue iff the cap is not reached and SOME element has |delta| > eps (all-NaN: none has)
    const bool cont = (st->iterations != a.max_iterations) && any_delta && (diff > a.eps);
    st->diff_bits = 0ull;
    if (!ok) st->error = 1;
    if (abort_all) st->aborted = 1;
    if (!cont || !ok || abort_all) st->done = 1;
  }
}

__global__ void barrier_kernel(const BarrierArgs b) {
  if (b.world <= 1) return;
  IterState *st = b.state;
  const unsigned long long seq = st->barrier_seq + 1;
  const bool ok = warp_barrier_exchange(b, seq, 0ull, 0.0);
  if ((threadIdx.x & 31) == 0) {
    st->barrier_seq = seq;
    if (!ok) {
      st->error = 1;
      st->done = 1;
    }
  }
}

// ---- normalise (:156-161): deterministic two-stage sum, then divide ----------------------------------

__global__ void __launch_bounds__(kBlockThreads) partial_sum_kernel(const double *rank, uint64_t count,
                                                                    double *partials) {
  // block b sums the contiguous chunk [b*chunk, (b+1)*chunk): thread-strided partials, fixed tree.
  const uint64_t chunk = (count + gridDim.x - 1) / gridDim.x;
  const uint64_t lo = chunk * blockIdx.x;
  const uint64_t hi = (lo + chunk < count) ? lo + chunk : count;
  double acc = 0.0;
  for (uint64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) acc += rank[i];
  __shared__ double sm[kBlockThreads];
  sm[threadIdx.x] = acc;
  __syncthreads();
  for (int o = kBlockThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sm[threadIdx.x] += sm[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) partials[blockIdx.x] = sm[0];
}

__global__ void final_sum_kernel(const double *partials, int count, const BarrierArgs b) {
  __shared__ double sm[kSumBlocks];
  for (int i = threadIdx.x; i < kSumBlocks; i += blockDim.x) sm[i] = i < count ? partials[i] : 0.0;
  __syncthreads();
  for (int o = kSumBlocks / 2; o > 0; o >>= 1) {
    for (int i = threadIdx.x; i < o; i += blockDim.x) sm[i] += sm[i + o];
    __syncthreads();
  }
  IterState *st = b.state;
  if (threadIdx.x < 32) {
    const double local = sm[0];
    double total = local;
    bool ok = true;
    unsigned long long seq = st->barrier_seq;
    if (b.world > 1) {
      seq += 1;
      ok = warp_barrier_exchange(b, seq, 0ull, local);
      total = 0.0;
      for (int q = 0; q < b.world; ++q) total += b.mine->rank_sum[seq & 1ull][q];  // same order everywhere
    }
    if (threadIdx.x == 0) {
      st->barrier_seq = seq;
      st->local_sum = local;
      st->rank_sum = total;
      if (!ok) st->error = 1;
    }
  }
}

__global__ void __launch_bounds__(kBlockThreads) write_original_order_kernel(uint64_t n, const uint32_t *label_of,
                                                                             const double *rank,
                                                                             const IterState *state, double *out) {
  const double sum = state->rank_sum;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n; v += stride)
    out[v] = __ddiv_rn(rank[label_of[v]], sum);  // :158-160
}

__global__ void __launch_bounds__(kBlockThreads) write_local_kernel(uint64_t local_rows, const double *rank,
                                                                    const uint32_t *local_vertex,
                                                                    const IterState *state, double *out,
                                                                    uint32_t *vertex_out) {
  const double sum = state->rank_sum;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t r = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < local_rows; r += stride) {
    out[r] = __ddiv_rn(rank[r], sum);
    if (vertex_out) vertex_out[r] = local_vertex[r];
  }
}

// ---- host-side launch helpers -------------------------------------------------------------------------

// a whole number of resident waves on the SMs; the occupancy query is made once per kernel per graph handle (not ~6
// driver calls per iteration)
int grid_for(const Graph &g, const void *kernel, int threads = kBlockThreads) {
  for (int i = 0; i < g.occ_cached; ++i)
    if (g.occ_kernel[i] == kernel) return g.sm_count * g.occ_blocks[i];
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0) != cudaSuccess || per_sm < 1) per_sm = 4;
  if (g.occ_cached < Graph::kOccSlots) {
    g.occ_kernel[g.occ_cached] = kernel;
    g.occ_blocks[g.occ_cached] = per_sm;
    ++g.occ_cached;
  }
  return g.sm_count * per_sm;
}

uint64_t ceil_div(uint64_t a, uint64_t b) { return (a + b - 1) / b; }

RowEpilogue make_epilogue(const Graph &g, uint64_t it, const IterateConfig &cfg) {
  RowEpilogue ep{};
  ep.base = (1.0 - cfg.damping) / static_cast<double>(g.n);
  ep.damping = cfg.damping;
  ep.rank = g.rank;
  ep.outdeg = g.outdeg_l;
  ep.map = g.map;
  ep.world = static_cast<int>(g.part_world);
  ep.self = static_cast<int>(g.part_rank);
  ep.need = reinterpret_cast<const uint8_t *>(g.need_mask);
  ep.store_mask = g.tun.lone_partition ? (1u << g.part_rank) : 0xFFFFFFFFu;
  const int out_parity = static_cast<int>((it + 1) & 1ull);
  for (int q = 0; q < kMaxPeers; ++q) ep.contrib_out[q] = q < ep.world ? g.peers.contrib[out_parity][q] : nullptr;
  return ep;
}

// Tunables are read from the environment once per graph (graph_build.cu, Graph::tun) -- no process-wide statics,
// so concurrent calls from several sessions never race on them.
GatherWindow make_window(const Graph &g) {
  const uint64_t hot_mb = g.tun.l2_hot_mb;
  const uint64_t total = std::min<uint64_t>((g.n + 1) * sizeof(double), 0xFFFFFF00ull);
  GatherWindow w{};
  w.total_bytes = static_cast<uint32_t>(total);
  w.hot_bytes = static_cast<uint32_t>(std::min<uint64_t>(total, hot_mb << 20));
  w.world = g.part_world;
  w.l1_hot = g.l1_hot_labels();
  w.l2_hot = g.l2_hot_labels();
  w.table_n = g.table_labels();
  // global-order labelling: "hot" is one label prefix on every partition -> the exact single-partition code
  w.path = g.idx_flagged ? kPathFlags
           : (g.tun.multi_aware && !g.map.global_order && (g.part_world > 1 || g.tun.force_multi_path)) ? kPathLookup
                                                                                                        : kPathRange;
  for (uint32_t q = 0; q < static_cast<uint32_t>(kMaxPeers); ++q)
    w.start[q] = q < g.part_world ? static_cast<uint32_t>(g.part_start[q]) : 0xFFFFFFFFu;
  return w;
}

// The only places that fill the gather kernels' arguments from a graph; `vec` is the gathered vector (slot n holds 0),
// `weighted` multiplies every gathered value by its edge weight (one partition only, see launch_gather_phase).
SellArgs make_sell_args(const Graph &g, const double *vec, const GatherWindow &window, bool weighted) {
  SellArgs s{};
  s.colbase = g.sell_colbase;
  s.idx = g.sell_idx;
  s.w = weighted ? g.sell_w : nullptr;
  s.work = g.sell_work_items;
  s.n_work = g.sell_work;
  s.queue = g.queue;
  s.mode = g.sell_static ? 1u : 0u;
  s.first_row = g.n_heavy;
  s.end_row = g.n_heavy + g.n_sell;
  s.contrib_in = vec;
  s.window = window;
  s.state = g.state;
  s.sums = g.sell_sums;
  s.stage_val = g.stage_val;
  return s;
}

HeavyArgs make_heavy_args(const Graph &g, const double *vec, const GatherWindow &window, bool weighted) {
  HeavyArgs h{};
  h.heavy_ptr = g.heavy_ptr;
  h.heavy_idx = g.heavy_idx;
  h.heavy_w = weighted ? g.heavy_w : nullptr;
  h.seg_row = g.seg_row;
  h.seg_begin = g.seg_begin;
  h.seg_slot = g.seg_slot;
  h.seg_first = g.seg_first;
  h.seg_partial = g.seg_partial;
  h.row_sums = g.heavy_sums;
  h.n_seg = g.n_cold_seg;
  h.n_heavy = g.n_heavy;
  h.segment_edges = g.segment_edges;
  h.contrib_in = vec;
  h.window = window;
  h.state = g.state;
  return h;
}

BarrierArgs make_barrier(const Graph &g) {
  BarrierArgs b{};
  b.state = g.state;
  b.mine = g.flags();
  b.rank = static_cast<int>(g.part_rank);
  b.world = static_cast<int>(g.part_world);
  for (int q = 0; q < kMaxPeers; ++q) b.peer[q] = q < b.world ? g.peers.flags[q] : nullptr;
  if (g.tun.lone_partition) {  // profiling: a barrier of one over the own flag page
    b.rank = 0;
    b.world = 1;
    for (int q = 0; q < kMaxPeers; ++q) b.peer[q] = q == 0 ? g.flags() : nullptr;
  }
  b.timeout_ns = g.tun.barrier_timeout_ms * 1000000ull;
  return b;
}

}  // namespace

ZeroRanges make_zero_ranges(const Graph &g) {
  ZeroRanges zr{};
  zr.world = static_cast<int>(g.part_world);
  for (int q = 0; q < kMaxPeers; ++q) {
    zr.lo[q] = q < zr.world ? g.zero_lo[q] : 0;
    zr.hi[q] = q < zr.world ? g.zero_hi[q] : 0;
  }
  return zr;
}

// the rank of a zero in-degree row once the loop has run at least once ((1-d)/N); 1/N if it never runs
double zero_row_rank(const Graph &g, const IterateConfig &cfg) {
  return cfg.max_iterations == 0 ? 1.0 / static_cast<double>(g.n) : (1.0 - cfg.damping) / static_cast<double>(g.n);
}

using SellKernel = void (*)(SellArgs);
static SellKernel plain_sell_kernel(uint32_t path) {
  return path == kPathFlags ? sell_rows_kernel<kPathFlags>
         : path == kPathLookup ? sell_rows_kernel<kPathLookup>
                               : sell_rows_kernel<kPathRange>;
}

int setup_sell_table_kernel(int device, uint32_t *bytes) {
  int optin = 0;
  MGB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  const void *const kernels[] = {reinterpret_cast<const void *>(sell_rows_table_kernel<kPathRange>),
                                 reinterpret_cast<const void *>(sell_rows_table_kernel<kPathFlags>)};
  size_t static_bytes = 0;
  for (const void *fn : kernels) {
    cudaFuncAttributes attr{};
    MGB_CUDA(cudaFuncGetAttributes(&attr, fn));
    static_bytes = std::max(static_bytes, attr.sharedSizeBytes);
  }
  const size_t room = static_cast<size_t>(optin) > static_bytes ? static_cast<size_t>(optin) - static_bytes : 0;
  *bytes = static_cast<uint32_t>(room / 16 * 16);
  // The dynamic shared memory limit is a property of the kernel on the device, shared by every graph handle of the
  // process: it is always raised to the device's largest table, never set to one handle's table size, which a
  // concurrent call with a larger table would then exceed at launch.  The carveout hint keeps the L1 / shared split at
  // the smallest shared part each launch's table needs (the L1 left over is what the walk's gathers land in).
  for (const void *fn : kernels) {
    MGB_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(*bytes)));
    MGB_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxL1));
  }
  return MGB200_OK;
}

int sell_warps_per_sm(const Graph &g) {
  const GatherWindow w = make_window(g);
  if (w.table_n > 0 && w.path != kPathLookup) return kTableThreads / 32;
  return grid_for(g, reinterpret_cast<const void *>(plain_sell_kernel(w.path))) / g.sm_count * kWarpsPerBlock;
}

// SELL rows: the plain kernel (MGB_SELL_MIN_BLOCKS x 256 threads per SM) or, with a hot table, one kTableThreads CTA per SM
int launch_sell_rows(Graph &g, const SellArgs &s) {
  const uint32_t table_n = s.window.table_n;
  if (s.w != nullptr) {
    if (s.window.path != kPathRange) {
      set_error("internal: weighted gathers exist for the single-partition range path only");
      return MGB200_ERR_INVALID_ARGUMENT;
    }
    const int grid = static_cast<int>(std::min(
        static_cast<uint64_t>(grid_for(g, reinterpret_cast<const void *>(sell_rows_weighted_kernel))),
        ceil_div(g.sell_work, kWarpsPerBlock)));
    sell_rows_weighted_kernel<<<grid, kBlockThreads, 0, g.stream>>>(s);
  } else if (table_n > 0 && s.window.path != kPathLookup) {
    void (*const fn)(SellArgs) = s.window.path == kPathFlags ? sell_rows_table_kernel<kPathFlags> : sell_rows_table_kernel<kPathRange>;
    const int bytes = static_cast<int>(table_n * sizeof(double));  // <= the limit setup_sell_table_kernel granted
    const int grid = static_cast<int>(std::min<uint64_t>(g.sm_count, ceil_div(g.sell_work, kTableThreads / 32)));
    fn<<<grid, kTableThreads, bytes, g.stream>>>(s);
  } else {
    const SellKernel sell_fn = plain_sell_kernel(s.window.path);
    const int grid = static_cast<int>(std::min(
        static_cast<uint64_t>(grid_for(g, reinterpret_cast<const void *>(sell_fn))), ceil_div(g.sell_work, kWarpsPerBlock)));
    sell_fn<<<grid, kBlockThreads, 0, g.stream>>>(s);
  }
  MGB_CUDA(cudaGetLastError());
  return MGB200_OK;
}

// The same SELL rows through the TMA index ring + LDGSTS gathers (opt-in MGB200_SELL_KERNEL=stream, sell_stream.cuh)
int launch_sell_stream(Graph &g, const SellArgs &s) {
  if (!g.stream_attr_set) {  // per device, so per graph handle
    MGB_CUDA(cudaFuncSetAttribute(sell_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kStreamSmemBytes));
    g.stream_attr_set = true;
  }
  SellStreamArgs t{};
  t.colbase = s.colbase;
  t.idx = s.idx;
  t.item_begin = g.sell_item_begin;
  t.n_items = g.sell_items;
  t.first_row = s.first_row;
  t.end_row = s.end_row;
  t.contrib_in = s.contrib_in;
  t.window = s.window;
  t.state = s.state;
  t.sums = s.sums;
  const int grid = static_cast<int>(std::min<uint64_t>(g.sm_count, ceil_div(g.sell_items, kStreamWarps)));
  sell_stream_kernel<<<grid, kStreamThreads, kStreamSmemBytes, g.stream>>>(t);
  MGB_CUDA(cudaGetLastError());
  return MGB200_OK;
}

// The block passes over `vec`, one launch per non-empty block, in block order on the main stream.  They also stage the
// SELL walk's values from their blocks, so every gather path launches them before the SELL rows.
int launch_block_passes(Graph &g, const double *vec, uint64_t *launches) {
  const uint64_t grid_cap = static_cast<uint64_t>(grid_for(g, reinterpret_cast<const void *>(cold_block_kernel)));
  for (size_t b = 0; b + 1 < g.block_slice_first.size(); ++b) {
    BlockArgs a{};
    a.idx = g.block_idx;
    a.colbase = g.bslice_colbase;
    a.slot = g.block_slot;
    a.slice_begin = g.block_slice_first[b];
    a.slice_end = g.block_slice_first[b + 1];
    a.block = vec + g.block_lo[b];
    const uint64_t tail = std::min<uint64_t>((g.n + 1 - g.block_lo[b]) * sizeof(double), 0xFFFFFF00ull);
    a.block_bytes = static_cast<uint32_t>(std::min<uint64_t>(g.block_labels * sizeof(double), tail));
    a.tail_bytes = static_cast<uint32_t>(tail);
    a.contrib_in = vec;
    a.seg_partial = g.seg_partial;
    a.state = g.state;
    a.stage_src = g.stage_src;
    a.stage_val = g.stage_val;
    a.stage_begin = g.stage_entries ? g.stage_first[b] : 0;
    a.stage_end = g.stage_entries ? g.stage_first[b + 1] : 0;
    const uint64_t want = std::max(ceil_div(a.slice_end - a.slice_begin, kWarpsPerBlock),
                                   ceil_div(a.stage_end - a.stage_begin, kBlockThreads * kStageUnroll));
    const int grid = static_cast<int>(std::min(grid_cap, want));
    cold_block_kernel<<<grid, kBlockThreads, 0, g.stream>>>(a);
    MGB_CUDA(cudaGetLastError());
    ++*launches;
  }
  return MGB200_OK;
}

// Heavy-row partials: the tile chunks (shared-memory reads, a 2-byte offset stream; one CTA per work item, one per SM,
// as a tile takes most of the SM's shared memory) and the cold segments (random HBM gathers) write disjoint partials
// and wait on different units, so with both present the cold segments run on a stream of their own next to the tile
// kernel, joined back before the caller's row sums.  The tile kernel goes first: its CTAs need half an SM each and
// would wait behind a full grid of segment CTAs.  The segment grid leaves `reserve_ctas` CTA slots to other kernels.
int launch_heavy_partials(Graph &g, const HeavyArgs &h, uint64_t reserve_ctas, uint64_t *launches) {
  void (*const seg_fn)(HeavyArgs) = h.heavy_w != nullptr           ? heavy_segments_kernel<kPathRange, true>
                                    : h.window.path == kPathFlags  ? heavy_segments_kernel<kPathFlags>
                                    : h.window.path == kPathLookup ? heavy_segments_kernel<kPathLookup>
                                                                   : heavy_segments_kernel<kPathRange>;
  uint64_t seg_grid_cap = static_cast<uint64_t>(grid_for(g, reinterpret_cast<const void *>(seg_fn)));
  if (seg_grid_cap > reserve_ctas) seg_grid_cap -= reserve_ctas;
  const bool fork = g.tile_slices > 0 && g.n_cold_seg > 0;
  if (fork) {  // before the tile kernel: the cold stream waits for the earlier work of the main stream only
    MGB_CUDA(cudaEventRecord(g.cold_fork_ev, g.stream));
    MGB_CUDA(cudaStreamWaitEvent(g.cold_stream, g.cold_fork_ev, 0));
  }
  if (g.tile_slices > 0) {
    const TileArgs t{g.tile_idx,   g.tslice_colbase, g.tslice_tile,     g.tile_slot,  g.tile_slice_first,
                     g.tile_base,  g.tile_load,      g.tile_work_begin, g.tile_work,  g.tile_queue,
                     g.tun.tile_labels, h.contrib_in, g.seg_partial,    g.state};
    const int bytes = static_cast<int>((g.tun.tile_labels + 1) * sizeof(double));
    if (g.tile_attr_bytes < bytes) {
      MGB_CUDA(cudaFuncSetAttribute(heavy_tiles_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
      g.tile_attr_bytes = bytes;
    }
    const uint32_t grid = std::min<uint32_t>(g.tile_work, static_cast<uint32_t>(g.sm_count));
    heavy_tiles_kernel<<<grid, kTileThreads, bytes, g.stream>>>(t);
    MGB_CUDA(cudaGetLastError());
    ++*launches;
  }
  if (g.n_cold_seg > 0) {
    cudaStream_t cs = fork ? g.cold_stream : g.stream;
    const int grid = static_cast<int>(std::min(seg_grid_cap, ceil_div(g.n_cold_seg, kWarpsPerBlock)));
    seg_fn<<<grid, kBlockThreads, 0, cs>>>(h);
    MGB_CUDA(cudaGetLastError());
    ++*launches;
    if (fork) {
      MGB_CUDA(cudaEventRecord(g.cold_join_ev, g.cold_stream));
      MGB_CUDA(cudaStreamWaitEvent(g.stream, g.cold_join_ev, 0));
    }
  }
  return MGB200_OK;
}

// per heavy row: its partials summed in segment order into h.row_sums
int launch_heavy_rowsums(Graph &g, const HeavyArgs &h) {
  const int grid = static_cast<int>(
      std::min(static_cast<uint64_t>(grid_for(g, reinterpret_cast<const void *>(heavy_rowsum_kernel))),
               ceil_div(g.n_heavy, kWarpsPerBlock)));
  heavy_rowsum_kernel<<<grid, kBlockThreads, 0, g.stream>>>(h);
  MGB_CUDA(cudaGetLastError());
  return MGB200_OK;
}

int launch_init(Graph &g, const IterateConfig &cfg) {
  MGB_CUDA(cudaSetDevice(g.device));
  const int grid = grid_for(g, reinterpret_cast<const void *>(init_kernel));
  init_kernel<<<grid, kBlockThreads, 0, g.stream>>>(g.n, g.local_rows, g.n_heavy + g.n_sell, zero_row_rank(g, cfg),
                                                     g.rank, g.outdeg_l, g.contrib(0), g.contrib(1),
                                                     make_zero_ranges(g), g.state);
  MGB_CUDA(cudaGetLastError());
  return MGB200_OK;
}

int launch_barrier(Graph &g) {
  if (g.part_world <= 1) return MGB200_OK;
  barrier_kernel<<<1, 32, 0, g.stream>>>(make_barrier(g));
  MGB_CUDA(cudaGetLastError());
  return MGB200_OK;
}

// One iteration.  Main stream: (iteration 1: zero-row contribution refresh) -> block passes + SELL rows (the sell_rows
// event class; without SELL rows the passes open the heavy_segments class) -> heavy partials (tiles, segments) ->
// heavy finish -> [join] -> iteration end.  Side stream: the SELL epilogue, forked after the SELL rows:
// it is the kernel that pushes contributions to the peer GPUs (NVLink-bound), so it overlaps with the
// heavy-row kernels (L2-gather-bound) instead of queueing behind them.  Every kernel returns immediately
// once state->done is set, so the host may enqueue iterations ahead of the convergence decision.
int launch_iteration(Graph &g, uint64_t it, const IterateConfig &cfg, uint64_t *launch_count,
                     uint64_t *spmv_count) {
  const RowEpilogue ep = make_epilogue(g, it, cfg);
  const double *contrib_in = g.contrib(static_cast<int>(it & 1ull));
  const GatherWindow window = make_window(g);
  uint64_t launches = 0;
  const bool timed = g.time_spmv && g.timed_launches < Graph::kMaxTimedLaunches;
  auto tick = [&](int cls, int edge, cudaStream_t st) -> cudaError_t {
    if (!timed) return cudaSuccess;
    return cudaEventRecord(g.kev[(g.timed_launches * Graph::kClasses + cls) * 2 + edge], st);
  };
  if (it == 1 && g.any_zero_rows) {
    MGB_CUDA(tick(Graph::kClsZero, 0, g.stream));
    zero_refresh_kernel<<<grid_for(g, reinterpret_cast<const void *>(zero_refresh_kernel)), kBlockThreads, 0,
                          g.stream>>>(zero_row_rank(g, cfg), g.outdeg_l, g.contrib(0), make_zero_ranges(g), g.state);
    MGB_CUDA(tick(Graph::kClsZero, 1, g.stream));
    ++launches;
  }
  bool forked = false;
  if (g.n_slices > 0) {
    const SellArgs s = make_sell_args(g, contrib_in, window, false);
    cudaStream_t es = g.overlap_epilogue ? g.stream2 : g.stream;
    MGB_CUDA(tick(Graph::kClsSell, 0, g.stream));
    int rc = launch_block_passes(g, contrib_in, &launches);  // with SELL rows: inside the sell_rows class
    if (rc) return rc;
    rc = (g.tun.stream_kernel && g.sell_items > 0) ? launch_sell_stream(g, s) : launch_sell_rows(g, s);
    if (rc) return rc;
    ++launches;
    MGB_CUDA(tick(Graph::kClsSell, 1, g.stream));
    // the epilogue (+ NVLink push to the peers) of the SELL rows runs on the side stream, next to the heavy-row kernels
    if (g.overlap_epilogue) {
      MGB_CUDA(cudaEventRecord(g.fork_ev, g.stream));
      MGB_CUDA(cudaStreamWaitEvent(g.stream2, g.fork_ev, 0));
      forked = true;
    }
    // Across GPUs this kernel IS the exchange (one NVLink store per peer per row): it is bound by the links, not by the
    // SMs, and it must run NEXT TO the heavy-row kernels, not before or after them.  A full grid (4 CTAs/SM x 63
    // registers) takes the whole register file, so the heavy kernel (8 CTAs/SM x 32 registers, also the whole file)
    // only starts when it drains, and push and heavy rows run in sequence.  A small grid (MGB200_PUSH_CTAS per SM, default 1) leaves 6 of the heavy kernel's 8
    // CTA slots free and keeps enough stores in flight to fill the links.
    uint64_t egrid_cap = static_cast<uint64_t>(grid_for(g, reinterpret_cast<const void *>(row_epilogue_kernel)));
    if (g.part_world > 1 && g.overlap_epilogue && g.tun.push_ctas > 0)
      egrid_cap = std::min<uint64_t>(egrid_cap, static_cast<uint64_t>(g.sm_count) * g.tun.push_ctas);
    // the tile kernel needs half an SM's register file next to it (512 threads x 64 registers): at its full grid the
    // epilogue would hold every SM until it drains and the tile kernel would start only then
    if (g.overlap_epilogue && g.tile_slices)
      egrid_cap = std::min<uint64_t>(egrid_cap, static_cast<uint64_t>(g.sm_count) * kTileEpiCtas);
    const int egrid = static_cast<int>(std::min(egrid_cap, ceil_div(g.n_sell, kBlockThreads * kEpiRows)));
    MGB_CUDA(tick(Graph::kClsSellEpi, 0, es));
    row_epilogue_kernel<<<egrid, kBlockThreads, 0, es>>>(s.first_row, s.end_row, g.sell_sums, g.state, ep);
    MGB_CUDA(tick(Graph::kClsSellEpi, 1, es));
    ++launches;
    if (forked) MGB_CUDA(cudaEventRecord(g.join_ev, g.stream2));
    if (spmv_count) *spmv_count += 1;
  }
  if (g.n_seg > 0) {
    const HeavyArgs h = make_heavy_args(g, contrib_in, window, false);
    // leave register-file room for the push kernel's CTAs (63 registers x 256 threads each) next to the segment kernel
    const uint64_t reserve_ctas =
        (forked && g.part_world > 1 && g.tun.push_ctas > 0) ? static_cast<uint64_t>(g.sm_count) * 2 : 0;
    MGB_CUDA(tick(Graph::kClsHeavySeg, 0, g.stream));
    int rc = g.n_slices > 0 ? MGB200_OK : launch_block_passes(g, contrib_in, &launches);  // without: heavy class
    if (rc) return rc;
    rc = launch_heavy_partials(g, h, reserve_ctas, &launches);
    if (rc) return rc;
    MGB_CUDA(tick(Graph::kClsHeavySeg, 1, g.stream));
    MGB_CUDA(tick(Graph::kClsHeavyFin, 0, g.stream));
    rc = launch_heavy_rowsums(g, h);
    if (rc) return rc;
    const int grid = static_cast<int>(
        std::min(static_cast<uint64_t>(grid_for(g, reinterpret_cast<const void *>(row_epilogue_kernel))),
                 ceil_div(g.n_heavy, kBlockThreads * kEpiRows)));
    row_epilogue_kernel<<<grid, kBlockThreads, 0, g.stream>>>(0, g.n_heavy, g.heavy_sums, g.state, ep);
    MGB_CUDA(tick(Graph::kClsHeavyFin, 1, g.stream));
    launches += 2;
  }
  if (forked) MGB_CUDA(cudaStreamWaitEvent(g.stream, g.join_ev, 0));
  IterEndArgs e{};
  e.bar = make_barrier(g);
  e.max_iterations = cfg.max_iterations;
  e.eps = cfg.eps;
  e.extra_diff_bits = 0ull;
  if (g.any_zero_rows) {
    // the zero rows are elements of the reference's stop test too: |(1-d)/N - 1/N| in iteration 0, exactly 0 afterwards
    const double zr = zero_row_rank(g, cfg);
    const double zd = it == 0 ? fabs(zr - 1.0 / static_cast<double>(g.n)) : fabs(zr - zr);
    if (zd >= 0.0) {  // NaN contributes nothing, like the per-row test; same bits + 1 encoding as the rows' deltas
      memcpy(&e.extra_diff_bits, &zd, sizeof(zd));
      e.extra_diff_bits += 1ull;
    }
  }
  MGB_CUDA(tick(Graph::kClsIterEnd, 0, g.stream));
  iter_end_kernel<<<1, 32, 0, g.stream>>>(e);
  MGB_CUDA(tick(Graph::kClsIterEnd, 1, g.stream));
  ++launches;
  MGB_CUDA(cudaGetLastError());
  if (timed) ++g.timed_launches;
  if (launch_count) *launch_count += launches;
  return MGB200_OK;
}

// The gather phase alone, over an arbitrary per-label vector vec_in[n + 1] (slot n must hold 0): SELL row sums into
// g.sell_sums, heavy segment partials into g.seg_partial (summed per row by the caller in segment order).  This is
// y = A^T x for the rows of this partition with PageRank's kernels and cache policies; other SpMV-shaped paths hang
// their own epilogue on it (Katz: omega_i = A^T omega_{i-1}, katz.cu).  Kernels return at once while state->done is set.
int launch_gather_phase(Graph &g, const double *vec_in, uint64_t *launch_count, bool heavy_row_sums, bool weighted) {
  uint64_t launches = 0;
  const GatherWindow window = make_window(g);
  if (weighted && (window.path != kPathRange || (g.n_slices > 0 && !g.sell_w) || (g.n_seg > 0 && !g.heavy_w))) {
    set_error("this graph handle carries no edge weights (or is partitioned)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  if (const int rc = launch_block_passes(g, vec_in, &launches)) return rc;  // they stage the SELL walk's values
  if (g.n_slices > 0) {
    const int rc = launch_sell_rows(g, make_sell_args(g, vec_in, window, weighted));
    if (rc) return rc;
    ++launches;
  }
  if (g.n_seg > 0) {
    const HeavyArgs h = make_heavy_args(g, vec_in, window, weighted);  // weighted graphs have no tile or block class
    int rc = launch_heavy_partials(g, h, 0, &launches);
    if (rc) return rc;
    if (heavy_row_sums) {
      rc = launch_heavy_rowsums(g, h);
      if (rc) return rc;
      ++launches;
    }
  }
  MGB_CUDA(cudaGetLastError());
  if (launch_count) *launch_count += launches;
  return MGB200_OK;
}

int launch_sum_and_exchange(Graph &g) {
  const int blocks = static_cast<int>(std::min<uint64_t>(kSumBlocks, g.local_rows ? ceil_div(g.local_rows, 4096) : 1));
  partial_sum_kernel<<<blocks, kBlockThreads, 0, g.stream>>>(g.rank, g.local_rows, g.sum_partials);
  final_sum_kernel<<<1, 256, 0, g.stream>>>(g.sum_partials, blocks, make_barrier(g));
  MGB_CUDA(cudaGetLastError());
  return MGB200_OK;
}

int launch_write_ranks_original_order(Graph &g, double *d_out) {
  if (g.n == 0) return MGB200_OK;
  const int grid = static_cast<int>(
      std::min(static_cast<uint64_t>(grid_for(g, reinterpret_cast<const void *>(write_original_order_kernel))),
          ceil_div(g.n, kBlockThreads)));
  write_original_order_kernel<<<grid, kBlockThreads, 0, g.stream>>>(g.n, g.label_of, g.rank, g.state, d_out);
  MGB_CUDA(cudaGetLastError());
  return MGB200_OK;
}

int launch_write_ranks_local(Graph &g, double *d_rank_out, uint32_t *d_vertex_out) {
  if (g.local_rows == 0) return MGB200_OK;
  const int grid = static_cast<int>(
      std::min(static_cast<uint64_t>(grid_for(g, reinterpret_cast<const void *>(write_local_kernel))),
          ceil_div(g.local_rows, kBlockThreads)));
  write_local_kernel<<<grid, kBlockThreads, 0, g.stream>>>(g.local_rows, g.rank, g.local_vertex, g.state,
                                                           d_rank_out, d_vertex_out);
  MGB_CUDA(cudaGetLastError());
  return MGB200_OK;
}

}  // namespace mgb200

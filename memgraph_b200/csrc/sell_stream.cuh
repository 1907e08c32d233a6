// memgraph_b200/csrc/sell_stream.cuh -- the SELL-32 rows as a decoupled, asynchronous stream.
// (included by pagerank_kernels.cu inside namespace mgb200::{anonymous}, after the shared helpers)
//
// An alternative to sell_rows_kernel, kept as the documented experiment (opt-in: MGB200_SELL_KERNEL=stream):
// each warp owns a CONTIGUOUS run of slices = one contiguous span of sell_idx, and two asynchronous stages run
// ahead of the arithmetic:
//   1. TMA   : cp.async.bulk streams the span's column indices (4 KiB = 32 columns per chunk) into a
//              per-warp shared-memory ring, completion on an mbarrier  (SASS: UBLKCP / SYNCS)
//   2. gather: every lane issues cp.async (LDGSTS) 8-byte copies contrib[idx] -> shared memory for a
//              batch of 8 columns per commit group, kVals batches deep, no registers held
//   3. reduce: the lane adds its own landed values in column order (fixed order => deterministic) and
//              stores the row sum at a slice boundary (the epilogue is sell_epilogue_kernel, as for the rows kernel)
// Parity-green.  It was slower than the LDG kernel at scale-26 on the GPU it was written for: the divergent 8-byte
// LDGSTS costs more per sector in L1TEX than LDG, and deeper rings make it worse.  On the H100 it runs within 1 % of
// the LDG kernel (DESIGN.md §4).
// The TMA ring is the right tool for the contiguous index stream; the gather is better left to LDG.
#pragma once

#ifndef MGB_STREAM_WARPS
#define MGB_STREAM_WARPS 8        // warps per CTA (1 CTA per SM: the rings take most of the shared memory)
#endif
#ifndef MGB_STREAM_IDX_STAGES
#define MGB_STREAM_IDX_STAGES 3   // index-ring depth, chunks of kChunkCols columns
#endif
#ifndef MGB_STREAM_VALS
#define MGB_STREAM_VALS 4         // gather batches in flight per warp
#endif

constexpr int kStreamWarps = MGB_STREAM_WARPS;
constexpr int kStreamThreads = kStreamWarps * 32;
constexpr int kChunkCols = 32;                        // columns per TMA chunk
constexpr int kChunkBytes = kChunkCols * kSliceRows * 4;  // 4 KiB
constexpr int kIdxStages = MGB_STREAM_IDX_STAGES;
constexpr int kBatchCols = 8;                         // columns per cp.async commit group
constexpr int kVals = MGB_STREAM_VALS;
constexpr int kBatchesPerChunk = kChunkCols / kBatchCols;
constexpr int kWarpIdxBytes = kIdxStages * kChunkBytes;
constexpr int kWarpValBytes = kVals * kBatchCols * kSliceRows * 8;
constexpr int kWarpSmemBytes = kWarpIdxBytes + kWarpValBytes;
constexpr int kStreamSmemBytes = kStreamWarps * kWarpSmemBytes;

struct SellStreamArgs {
  const uint64_t *colbase;     // [n_slices + 1]
  const uint32_t *idx;         // SELL index array
  const uint64_t *item_begin;  // [n_items + 1] first slice of each work item (contiguous slice runs)
  uint32_t n_items;
  uint64_t first_row;
  uint64_t end_row;
  const double *contrib_in;
  GatherWindow window;
  IterState *state;
  double *sums;  // [n_sell] per-row sums, consumed by sell_epilogue_kernel
};

// Per-lane asynchronous 8-byte gather global -> shared (LDGSTS), with the gather window's L2 policy.
__device__ __forceinline__ void gather_async_8(uint32_t dst_smem, const double *src, uint64_t pol) {
#if MGB_GATHER_POLICY
  asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 8, %2;" ::"r"(dst_smem), "l"(src), "l"(pol)
               : "memory");
#else
  (void)pol;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst_smem), "l"(src) : "memory");
#endif
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

__global__ void __launch_bounds__(kStreamThreads, 1) sell_stream_kernel(const SellStreamArgs a) {
  extern __shared__ __align__(128) unsigned char stream_smem[];
  __shared__ __align__(8) unsigned long long full_bar[kStreamWarps][kIdxStages];
  if (ld_volatile_int(&a.state->done)) return;
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  unsigned char *my_smem = stream_smem + wib * kWarpSmemBytes;
  const uint32_t *idx_ring = reinterpret_cast<const uint32_t *>(my_smem);
  const double *val_ring = reinterpret_cast<const double *>(my_smem + kWarpIdxBytes);
  const uint32_t idx_ring_s = smem_u32(my_smem);
  const uint32_t val_ring_s = smem_u32(my_smem + kWarpIdxBytes);
  uint32_t bar_s[kIdxStages];
#pragma unroll
  for (int i = 0; i < kIdxStages; ++i) bar_s[i] = smem_u32(&full_bar[wib][i]);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < kIdxStages; ++i) mbar_init(bar_s[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  const uint64_t pol = make_evict_first_policy();
  const uint64_t gpol = make_gather_policy(a.contrib_in, a.window).hot;
  const uint32_t warps_total = gridDim.x * kStreamWarps;
  uint32_t chunks_done = 0;  // chunks consumed so far by this warp over all items (drives slot/parity)

  for (uint32_t item = blockIdx.x * kStreamWarps + wib; item < a.n_items; item += warps_total) {
    const uint64_t s_begin = a.item_begin[item], s_end = a.item_begin[item + 1];
    if (s_begin >= s_end) continue;
    const uint64_t cb = a.colbase[s_begin], ce = a.colbase[s_end];
    const uint64_t ncols = ce - cb;
    const uint32_t nchunks = static_cast<uint32_t>((ncols + kChunkCols - 1) / kChunkCols);
    const uint32_t nbatches = static_cast<uint32_t>((ncols + kBatchCols - 1) / kBatchCols);
    const unsigned char *span = reinterpret_cast<const unsigned char *>(a.idx) + cb * (kSliceRows * 4);

    auto issue_chunk = [&](uint32_t chunk) {  // lane 0 only
      const uint32_t g = chunks_done + chunk;  // global chunk counter of this warp
      const uint32_t slot = g % kIdxStages;
      const uint64_t first_col = static_cast<uint64_t>(chunk) * kChunkCols;
      const uint64_t cols = (ncols - first_col < kChunkCols) ? ncols - first_col : kChunkCols;
      const uint32_t bytes = static_cast<uint32_t>(cols) * (kSliceRows * 4);
      mbar_expect_tx(bar_s[slot], bytes);
      tma_load_1d(idx_ring_s + slot * kChunkBytes, span + first_col * (kSliceRows * 4), bytes, bar_s[slot], pol);
    };
    // prologue: fill the index ring
    if (lane == 0) {
      for (uint32_t c = 0; c < nchunks && c < static_cast<uint32_t>(kIdxStages); ++c) issue_chunk(c);
    }

    // issue one batch of gathers (columns [8b, 8b+8) of the span); always commits a group
    auto issue_batch = [&](uint32_t b) {
      if (b < nbatches) {
        const uint32_t chunk = b / kBatchesPerChunk;
        const uint32_t g = chunks_done + chunk;
        const uint32_t slot = g % kIdxStages;
        if (b % kBatchesPerChunk == 0) mbar_wait(bar_s[slot], (g / kIdxStages) & 1u);
        const uint32_t *src_idx = idx_ring + slot * (kChunkBytes / 4) + (b % kBatchesPerChunk) * (kBatchCols * kSliceRows) + lane;
        const uint32_t dst = val_ring_s + ((b % kVals) * (kBatchCols * kSliceRows) + lane) * 8;
        const uint64_t col0 = static_cast<uint64_t>(b) * kBatchCols;
#pragma unroll
        for (int j = 0; j < kBatchCols; ++j) {
          if (col0 + j < ncols) gather_async_8(dst + j * (kSliceRows * 8), a.contrib_in + src_idx[j * kSliceRows], gpol);
        }
        // last batch of a chunk: every lane has read the slot -> refill it with the chunk kIdxStages ahead
        if (b % kBatchesPerChunk == kBatchesPerChunk - 1 || b == nbatches - 1) {
          __syncwarp();
          if (lane == 0 && chunk + kIdxStages < nchunks) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            issue_chunk(chunk + kIdxStages);
          }
        }
      }
      cp_async_commit();
    };

    // slice bookkeeping: lane l caches colbase[block + l + 1] for a block of 32 slices
    uint64_t s = s_begin;
    uint64_t s_block = s_begin;
    uint64_t ends = (s_block + lane + 1 <= s_end) ? a.colbase[s_block + lane + 1] : ce;
    uint64_t slice_end = __shfl_sync(kFull, ends, 0) - cb;  // relative to the span
    double acc = 0.0;

#pragma unroll 1
    for (uint32_t b = 0; b < static_cast<uint32_t>(kVals - 1); ++b) issue_batch(b);
#pragma unroll 1
    for (uint32_t b = 0; b < nbatches; ++b) {
      issue_batch(b + kVals - 1);
      cp_async_wait<kVals - 1>();
      const double *v = val_ring + (b % kVals) * (kBatchCols * kSliceRows) + lane;
      const uint64_t col0 = static_cast<uint64_t>(b) * kBatchCols;
#pragma unroll
      for (int j = 0; j < kBatchCols; ++j) {
        const uint64_t col = col0 + j;
        if (col < ncols) {
          acc += v[j * kSliceRows];
          if (col + 1 == slice_end) {
            const uint64_t row = a.first_row + s * kSliceRows + lane;
            if (row < a.end_row) a.sums[row - a.first_row] = acc;
            acc = 0.0;
            ++s;
            if (s < s_end) {
              if (s - s_block == 32) {
                s_block = s;
                ends = (s_block + lane + 1 <= s_end) ? a.colbase[s_block + lane + 1] : ce;
              }
              slice_end = __shfl_sync(kFull, ends, static_cast<int>(s - s_block)) - cb;
            }
          }
        }
      }
    }
    cp_async_wait<0>();
    __syncwarp();
    chunks_done += nchunks;
  }
}

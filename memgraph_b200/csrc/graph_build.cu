// memgraph_b200/csrc/graph_build.cu -- COO on the device -> degree-sorted SELL-32 + segmented CSC.
//
// This is the device-side counterpart of the reference's graph constructors
// (PageRankGraph(n, m, edges), pagerank.cpp:165-181; CreatePageRankGraph, pagerank_module.cpp:18-54):
// they produce a source-ordered edge list plus out-degrees for a CPU push loop; this produces the
// pull layout the sm_90a kernels stream.  It runs once per graph and is outside the timed
// iteration (SURVEY 8d); sorting and scanning use CUB (library code, like cuBLAS for a plain GEMM),
// the layout kernels are ours.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cub/cub.cuh>
#include <vector>

#include "core.hpp"

namespace mgb200 {
namespace {

// ---- degrees ----------------------------------------------------------------------------------------

__global__ void degree_kernel(uint64_t m, uint64_t n, const uint32_t *from, const uint32_t *to, uint32_t *outdeg,
                              uint32_t *indeg, int *bad) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t e = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < m; e += stride) {
    const uint32_t s = from[e], d = to[e];
    if (s >= n || d >= n) {
      *bad = 1;
      continue;
    }
    atomicAdd(outdeg + s, 1u);
    atomicAdd(indeg + d, 1u);
  }
}

// sort key: in-degree descending, then out-degree descending (stable sort keeps original id order)
__global__ void sort_key_kernel(uint64_t n, const uint32_t *indeg, const uint32_t *outdeg, uint64_t *key,
                                uint32_t *id) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n; v += stride) {
    key[v] = (static_cast<uint64_t>(~indeg[v]) << 32) | static_cast<uint64_t>(~outdeg[v]);
    id[v] = static_cast<uint32_t>(v);
  }
}

struct Dealer {  // sorted position -> global label when positions are dealt round-robin to P owners
  uint64_t n;
  uint32_t world;
  __host__ __device__ uint64_t count(uint32_t q) const { return (n + world - 1 - q) / world; }
  __host__ __device__ uint64_t start(uint32_t q) const {
    // sum_{r<q} count(r): the first (n % world) owners hold one extra row
    const uint64_t base = n / world, extra = n % world;
    return static_cast<uint64_t>(q) * base + (q < extra ? q : extra);
  }
  __host__ __device__ uint64_t label(uint64_t pos) const {
    const uint32_t owner = static_cast<uint32_t>(pos % world);
    return start(owner) + pos / world;
  }
};

__global__ void label_kernel(RowMap map, const uint32_t *sorted_id, const uint32_t *indeg, const uint32_t *outdeg,
                             uint32_t *label_of, uint32_t *indeg_l, uint32_t *outdeg_l, uint32_t *vertex_of_label) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t pos = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; pos < map.n; pos += stride) {
    const uint32_t v = sorted_id[pos];
    const uint64_t l = map.label_of_pos(pos);
    label_of[v] = static_cast<uint32_t>(l);
    indeg_l[l] = indeg[v];
    outdeg_l[l] = outdeg[v];
    vertex_of_label[l] = v;
  }
}

// ---- edges owned by this partition -> (local row, source label) keys ---------------------------------

__global__ void edge_key_all_kernel(uint64_t m, const uint32_t *from, const uint32_t *to, const uint32_t *label_of,
                                    uint64_t *key) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t e = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < m; e += stride)
    key[e] = (static_cast<uint64_t>(label_of[to[e]]) << 32) | label_of[from[e]];
}

__global__ void out_weight_kernel(uint64_t m, const uint32_t *from, const double *w, const uint32_t *label_of, double *outw_l) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t e = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < m; e += stride)
    atomicAdd(outw_l + label_of[from[e]], w[e]);
}

__global__ void edge_key_owned_kernel(uint64_t m, const uint32_t *from, const uint32_t *to, const uint32_t *label_of,
                                      RowMap map, uint64_t row_hi, uint64_t *key,
                                      unsigned long long *cursor) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const int lane = threadIdx.x & 31;
  const uint64_t m_round = (m + 31) / 32 * 32;  // keep whole warps in the loop for the ballot
  for (uint64_t e = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < m_round; e += stride) {
    uint64_t dl = 0;
    bool mine = false;
    if (e < m) {
      dl = label_of[to[e]];
      mine = map.global_order ? map.owner(dl) == map.rank : (dl >= map.row_lo && dl < row_hi);
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, mine);
    if (ballot == 0) continue;
    unsigned long long base = 0;
    if (lane == __ffs(ballot) - 1) base = atomicAdd(cursor, static_cast<unsigned long long>(__popc(ballot)));
    base = __shfl_sync(0xffffffffu, base, __ffs(ballot) - 1);
    if (mine) {
      const unsigned before = __popc(ballot & ((1u << lane) - 1u));
      const uint64_t local = map.global_order ? map.local_of(dl) : dl - map.row_lo;
      key[base + before] = (local << 32) | label_of[from[e]];
    }
  }
}

// ---- class boundaries: rows are sorted by in-degree descending ----------------------------------------

__global__ void class_count_kernel(uint64_t rows, const uint32_t *indeg_local, uint32_t heavy_min,
                                   unsigned long long *counts /* [0]=heavy, [1]=nonzero, [2]=edges */) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  unsigned long long h = 0, nz = 0, ed = 0;
  for (uint64_t r = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < rows; r += stride) {
    const uint32_t d = indeg_local[r];
    h += d >= heavy_min;
    nz += d > 0;
    ed += d;
  }
  for (int o = 16; o > 0; o >>= 1) {
    h += __shfl_xor_sync(0xffffffffu, h, o);
    nz += __shfl_xor_sync(0xffffffffu, nz, o);
    ed += __shfl_xor_sync(0xffffffffu, ed, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (h) atomicAdd(counts + 0, h);
    if (nz) atomicAdd(counts + 1, nz);
    if (ed) atomicAdd(counts + 2, ed);
  }
}

// non-zero in-degree rows per partition: label l belongs to the partition whose [start, start+count) holds it
__global__ void nonzero_per_partition_kernel(Dealer deal, const uint32_t *indeg_l, unsigned long long *nz) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint32_t q = 0; q < deal.world; ++q) {
    const uint64_t lo = deal.start(q), hi = lo + deal.count(q);
    unsigned long long c = 0;
    for (uint64_t l = lo + static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; l < hi; l += stride)
      c += indeg_l[l] > 0;
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(nz + q, c);
  }
}

// Which partitions gather the contribution of an owned row?  Every partition sees the whole edge list, so this is local
// work: edge u -> v makes owner(v) a reader of u.  At P = 8 on RMAT only 48 % of the (vertex, peer) pairs are readers
// (scripts/push_need.py): the other half of the NVLink pushes is never looked at.
__global__ void need_mask_kernel(uint64_t m, const uint32_t *from, const uint32_t *to, const uint32_t *label_of,
                                 RowMap map, uint32_t *words) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t e = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < m; e += stride) {
    const uint64_t ul = label_of[from[e]];
    if (map.owner(ul) != map.rank) continue;
    const uint32_t q = map.owner(label_of[to[e]]);
    if (q == map.rank) continue;
    const uint64_t row = map.local_of(ul);
    const uint32_t bit = (1u << q) << ((row & 3u) * 8u);
    uint32_t *w = words + (row >> 2);
    if ((*reinterpret_cast<volatile uint32_t *>(w) & bit) == 0) atomicOr(w, bit);  // hubs: one atomic, then reads
  }
}

struct U32ToU64 {
  __host__ __device__ uint64_t operator()(uint32_t v) const { return v; }
};

// ---- heavy class ---------------------------------------------------------------------------------------

// Hotness of a source label (core.hpp kIdxL2Hot / kIdxL1Hot), decided once per stored index instead of once per
// gather per iteration: local = label - first label of the owning partition (the dealt labelling gives every
// partition's range its own hottest-first order), compared with the thresholds the gather window uses.
struct IndexFlags {
  Dealer deal;
  uint32_t l1_hot, l2_hot;  // Graph::l1_hot_labels() (kNoL1Hints -> no L1 flag is ever read), l2_hot_labels()
  uint32_t enabled;
  uint32_t table_per_owner;  // > 0: the hottest labels of every owner live in the SELL kernel's shared-memory table;
                             // their stored index is code 01 in bits 31/30 + the table slot (owner * per_owner + local)
  __device__ uint32_t operator()(uint32_t label) const {
    if (!enabled) return label;
    if (label >= deal.n) return label | kIdxL2Hot | kIdxL1Hot;  // the pad slot: one address, read by every slice
    uint32_t s0 = 0, owner = 0;
    for (uint32_t q = 1; q < deal.world; ++q) {
      const uint32_t s = static_cast<uint32_t>(deal.start(q));
      if (label >= s) {
        s0 = s;
        owner = q;
      }
    }
    const uint32_t local = label - s0;
    if (local < table_per_owner) return kIdxL1Hot | (owner * table_per_owner + local);
    const bool l2 = local < l2_hot;
    // with a table, code 01 means "table slot", so a label outside the L2 window (L2_HOT_MB=0, or an L1 window larger
    // than the L2 one) keeps no L1 flag: L1-hot without L2-hot would read as a slot
    const bool l1 = l1_hot != kNoL1Hints && local < l1_hot && (l2 || table_per_owner == 0);
    return label | (l2 ? kIdxL2Hot : 0u) | (l1 ? kIdxL1Hot : 0u);
  }
};

__global__ void low32_kernel(uint64_t count, const uint64_t *key, IndexFlags flags, uint32_t *out) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t e = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < count; e += stride)
    out[e] = flags(static_cast<uint32_t>(key[e]));
}

// Which sources a heavy row gathers from shared-memory tiles: every owner's first `hot` labels (local label below
// `hot`, like the L2 window's hot_divisor()) -- P owners under the dealt labelling, else one owner whose range is [0, n).
// It depends on the labelling and the MGB200_TILE_* knobs only, never on the cache-policy knobs.
struct TileSet {
  Dealer owners;
  uint64_t hot;
  __device__ bool hot_label(uint32_t label) const {
    uint64_t s0 = 0;
    for (uint32_t q = 1; q < owners.world; ++q)
      if (label >= owners.start(q)) s0 = owners.start(q);
    return label - s0 < hot;
  }
};
struct ColdKey {  // cub::DeviceSelect predicate: the edge's source is neither tiled nor in the block class
  TileSet ts;
  uint64_t block_from;  // first label of the block class (n + 1 without one)
  __device__ bool operator()(uint64_t key) const {
    const uint32_t src = static_cast<uint32_t>(key);
    return src < block_from && !ts.hot_label(src);
  }
};
struct BlockKey {  // cub::DeviceSelect predicate: the edge's source is in the block class
  uint64_t block_from;
  __device__ bool operator()(uint64_t key) const { return static_cast<uint32_t>(key) >= block_from; }
};

__device__ __forceinline__ uint64_t lower_bound_key(const uint64_t *key, uint64_t lo, uint64_t hi, uint64_t v) {
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (key[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// (heavy row r, tile t) pairs, p = r * n_tiles + t: edges of r whose source lies in [tile_lo[t], tile_hi[t]) -- one
// contiguous run of the row's ascending sources -- and the chunks of at most `chunk` edges they make
__global__ void tile_pair_kernel(uint64_t n_heavy, uint32_t n_tiles, const uint64_t *row_ptr, const uint64_t *key,
                                 const uint32_t *tile_lo, const uint32_t *tile_hi, uint32_t chunk, uint32_t *pair_cnt,
                                 uint64_t *pair_chunks, unsigned long long *tile_chunks) {
  const uint64_t pairs = n_heavy * n_tiles;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t p = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; p < pairs; p += stride) {
    const uint64_t r = p / n_tiles;
    const uint32_t t = static_cast<uint32_t>(p % n_tiles);
    const uint64_t e1 = row_ptr[r + 1];
    const uint64_t lo = lower_bound_key(key, row_ptr[r], e1, (r << 32) | tile_lo[t]);
    const uint64_t cnt = lower_bound_key(key, lo, e1, (r << 32) | tile_hi[t]) - lo;
    const uint64_t nch = (cnt + chunk - 1) / chunk;
    pair_cnt[p] = static_cast<uint32_t>(cnt);
    pair_chunks[p] = nch;
    if (nch) atomicAdd(tile_chunks + t, static_cast<unsigned long long>(nch));
  }
}

// per heavy row: cold in-degree and tile chunks (no tiles: the in-degree and 0)
__global__ void tile_row_kernel(uint64_t n_heavy, uint32_t n_tiles, const uint32_t *indeg_local, const uint32_t *pair_cnt,
                                const uint64_t *pair_chunks, const uint64_t *block_ptr, uint64_t *cold_deg,
                                uint64_t *row_chunks) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t r = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < n_heavy; r += stride) {
    uint64_t hot = 0, chunks = 0;
    for (uint32_t t = 0; t < n_tiles; ++t) {
      hot += pair_cnt[r * n_tiles + t];
      chunks += pair_chunks[r * n_tiles + t];
    }
    cold_deg[r] = indeg_local[r] - hot - (block_ptr ? block_ptr[r + 1] - block_ptr[r] : 0);  // block edges excluded
    row_chunks[r] = chunks;
  }
}

// block chunks of local row r: [chunk_first[block_ptr[r]], chunk_first[block_ptr[r + 1]])
__device__ __forceinline__ uint64_t row_block_chunks(const uint64_t *block_ptr, const uint64_t *chunk_first, uint64_t r) {
  return block_ptr ? chunk_first[block_ptr[r + 1]] - chunk_first[block_ptr[r]] : 0;
}

// per heavy row: partials (tile chunks + cold segments + block chunks) and cold segments
__global__ void seg_count_kernel(uint64_t n_heavy, const uint64_t *cold_deg, const uint64_t *row_chunks,
                                 const uint64_t *block_ptr, const uint64_t *block_chunk_first, uint32_t seg_edges,
                                 uint64_t *row_parts, uint64_t *row_cold_segs) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t r = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < n_heavy; r += stride) {
    const uint64_t segs = (cold_deg[r] + seg_edges - 1) / seg_edges;
    row_parts[r] = row_chunks[r] + segs + row_block_chunks(block_ptr, block_chunk_first, r);
    row_cold_segs[r] = segs;
  }
}

// one record per tile chunk, in row order (= partial order): sort key (tile, length descending), first edge, partial
__global__ void tile_chunk_kernel(uint64_t n_heavy, uint32_t n_tiles, const uint64_t *row_ptr, const uint64_t *key,
                                  const uint32_t *tile_lo, const uint32_t *pair_cnt, const uint64_t *pair_chunk_first,
                                  const uint64_t *seg_first, uint32_t chunk, uint64_t *chunk_key, uint64_t *chunk_id,
                                  uint64_t *chunk_begin, uint32_t *chunk_len, uint64_t *chunk_slot) {
  const uint64_t pairs = n_heavy * n_tiles;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t p = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; p < pairs; p += stride) {
    const uint32_t cnt = pair_cnt[p];
    if (cnt == 0) continue;
    const uint64_t r = p / n_tiles;
    const uint32_t t = static_cast<uint32_t>(p % n_tiles);
    const uint64_t lo = lower_bound_key(key, row_ptr[r], row_ptr[r + 1], (r << 32) | tile_lo[t]);
    const uint64_t c0 = pair_chunk_first[p], row_c0 = pair_chunk_first[r * n_tiles];
    for (uint32_t k = 0; k * static_cast<uint64_t>(chunk) < cnt; ++k) {
      const uint64_t c = c0 + k;
      const uint32_t len = static_cast<uint32_t>(min(static_cast<uint64_t>(chunk), cnt - static_cast<uint64_t>(k) * chunk));
      chunk_key[c] = (static_cast<uint64_t>(t) << 32) | (0xFFFFFFFFu - len);
      chunk_id[c] = c;
      chunk_begin[c] = lo + static_cast<uint64_t>(k) * chunk;
      chunk_len[c] = len;
      chunk_slot[c] = seg_first[r] + (c - row_c0);
    }
  }
}

// width of every tile slice = length of its first (longest) chunk
__global__ void tile_width_kernel(uint64_t n_slices, const uint32_t *slice_tile, const uint64_t *tile_slice_first,
                                  const uint64_t *tile_chunk_first, const uint64_t *sorted_id, const uint32_t *chunk_len,
                                  uint64_t *width) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t s = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; s < n_slices; s += stride) {
    const uint32_t t = slice_tile[s];
    width[s] = chunk_len[sorted_id[tile_chunk_first[t] + (s - tile_slice_first[t]) * kSliceRows]];
  }
}

// one warp per tile slice, lane l = chunk l of the slice: its offsets column-major, padded with `pad` (slot T = 0.0)
__global__ void tile_fill_kernel(uint64_t n_slices, const uint32_t *slice_tile, const uint64_t *tile_slice_first,
                                 const uint64_t *tile_chunk_first, const uint32_t *tile_base, const uint64_t *colbase,
                                 const uint64_t *sorted_id, const uint64_t *chunk_begin, const uint32_t *chunk_len,
                                 const uint64_t *chunk_slot, const uint64_t *key, uint16_t pad, uint16_t *tile_idx,
                                 uint64_t *tile_slot) {
  const int lane = threadIdx.x & 31;
  const uint64_t warps_total = static_cast<uint64_t>(gridDim.x) * (blockDim.x >> 5);
  for (uint64_t s = static_cast<uint64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); s < n_slices;
       s += warps_total) {
    const uint32_t t = slice_tile[s];
    const uint64_t p = tile_chunk_first[t] + (s - tile_slice_first[t]) * kSliceRows + lane;
    const bool valid = p < tile_chunk_first[t + 1];
    uint64_t begin = 0, slot = ~0ull;
    uint32_t len = 0;
    if (valid) {
      const uint64_t c = sorted_id[p];
      begin = chunk_begin[c];
      len = chunk_len[c];
      slot = chunk_slot[c];
    }
    const uint64_t c0 = colbase[s];
    const uint32_t width = static_cast<uint32_t>(colbase[s + 1] - c0);
    const uint32_t base = tile_base[t];
    uint16_t *dst = tile_idx + c0 * kSliceRows + lane;
    for (uint32_t k = 0; k < width; ++k)
      dst[static_cast<size_t>(k) * kSliceRows] = k < len ? static_cast<uint16_t>(static_cast<uint32_t>(key[begin + k]) - base) : pad;
    tile_slot[s * kSliceRows + lane] = slot;
  }
}

__global__ void segment_fill_kernel(uint64_t n_heavy, const uint64_t *heavy_ptr, const uint64_t *cold_seg_first,
                                    uint32_t seg_edges, const uint64_t *seg_first, const uint64_t *block_ptr,
                                    const uint64_t *block_chunk_first, uint32_t *seg_row, uint64_t *seg_begin,
                                    uint64_t *seg_slot) {
  // one warp per heavy row; lanes stride over that row's cold segments, which follow its tile chunks and precede its
  // block chunks in partial order
  const int lane = threadIdx.x & 31;
  const uint64_t warps_total = static_cast<uint64_t>(gridDim.x) * (blockDim.x >> 5);
  for (uint64_t r = static_cast<uint64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n_heavy;
       r += warps_total) {
    const uint64_t s0 = cold_seg_first[r], s1 = cold_seg_first[r + 1], e0 = heavy_ptr[r];
    const uint64_t end = seg_first[r + 1] - row_block_chunks(block_ptr, block_chunk_first, r);
    for (uint64_t s = s0 + lane; s < s1; s += 32) {
      seg_row[s] = static_cast<uint32_t>(r);
      seg_begin[s] = e0 + (s - s0) * seg_edges;
      if (seg_slot) seg_slot[s] = end - (s1 - s);
    }
  }
}

// ---- SELL class ------------------------------------------------------------------------------------------

__global__ void slice_width_kernel(uint64_t n_slices, const uint32_t *indeg_local, uint64_t first_row,
                                   uint64_t *width) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t s = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; s < n_slices; s += stride)
    width[s] = indeg_local[first_row + s * kSliceRows];  // rows sorted descending: lane 0 is the widest
}

__global__ void sell_fill_kernel(uint64_t n_slices, uint64_t first_row, uint64_t end_row, const uint64_t *row_ptr,
                                 const uint64_t *key, const uint64_t *colbase, uint32_t pad, IndexFlags flags,
                                 uint32_t *sell_idx, const double *w_sorted, double *sell_w) {
  const int lane = threadIdx.x & 31;
  const uint64_t warps_total = static_cast<uint64_t>(gridDim.x) * (blockDim.x >> 5);
  for (uint64_t s = static_cast<uint64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); s < n_slices;
       s += warps_total) {
    const uint64_t c0 = colbase[s];
    const uint32_t width = static_cast<uint32_t>(colbase[s + 1] - c0);
    const uint64_t row = first_row + s * kSliceRows + lane;
    uint64_t e0 = 0;
    uint32_t deg = 0;
    if (row < end_row) {
      e0 = row_ptr[row];
      deg = static_cast<uint32_t>(row_ptr[row + 1] - e0);
    }
    uint32_t *dst = sell_idx + c0 * kSliceRows + lane;
    for (uint32_t k = 0; k < width; ++k)
      dst[static_cast<size_t>(k) * kSliceRows] = flags(k < deg ? static_cast<uint32_t>(key[e0 + k]) : pad);
    if (sell_w) {
      double *wd = sell_w + c0 * kSliceRows + lane;
      for (uint32_t k = 0; k < width; ++k) wd[static_cast<size_t>(k) * kSliceRows] = k < deg ? w_sorted[e0 + k] : 0.0;
    }
  }
}

// ---- block class ------------------------------------------------------------------------------------------

// per heavy row: the number of block edges (the tail of its ascending sources from `from` on)
__global__ void block_row_kernel(uint64_t rows, const uint64_t *row_ptr, const uint64_t *key, uint64_t from,
                                 uint64_t *block_cnt) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t r = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < rows; r += stride)
    block_cnt[r] = row_ptr[r + 1] - lower_bound_key(key, row_ptr[r], row_ptr[r + 1], (r << 32) | from);
}

// 1 where a block edge (compacted keys, row-major, ascending sources) starts a chunk: every `chunk`-th edge of a
// row's run of sources in one block
__global__ void block_start_kernel(uint64_t count, const uint64_t *bkey, const uint64_t *block_ptr, uint64_t from,
                                   uint64_t labels, uint32_t chunk, uint64_t *start) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += stride) {
    const uint64_t k = bkey[i], r = k >> 32, b = (static_cast<uint32_t>(k) - from) / labels;
    const uint64_t first = block_ptr[r];
    bool st = i == first || (static_cast<uint32_t>(bkey[i - 1]) - from) / labels != b;
    if (!st) st = (i - lower_bound_key(bkey, first, i, (r << 32) | (from + b * labels))) % chunk == 0;
    start[i] = st;
  }
}

// one record per chunk, in (row, block) order: first edge, row, per-block count
__global__ void block_chunk_kernel(uint64_t count, const uint64_t *bkey, const uint64_t *start, const uint64_t *chunk_of,
                                   uint64_t from, uint64_t labels, uint64_t *cbegin, uint32_t *crow,
                                   unsigned long long *per_block) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += stride) {
    if (!start[i]) continue;
    const uint64_t c = chunk_of[i], k = bkey[i];
    cbegin[c] = i;
    crow[c] = static_cast<uint32_t>(k >> 32);
    atomicAdd(per_block + (static_cast<uint32_t>(k) - from) / labels, 1ull);
  }
}

// chunk length and sort key (block, length descending); a stable sort keeps row order among equal keys
__global__ void block_len_kernel(uint64_t chunks, uint64_t count, const uint64_t *bkey, const uint64_t *cbegin,
                                 uint64_t from, uint64_t labels, uint32_t *clen, uint64_t *ckey, uint64_t *cid) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t c = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; c < chunks; c += stride) {
    const uint64_t b0 = cbegin[c];
    const uint32_t len = static_cast<uint32_t>((c + 1 < chunks ? cbegin[c + 1] : count) - b0);
    const uint64_t b = (static_cast<uint32_t>(bkey[b0]) - from) / labels;
    clen[c] = len;
    ckey[c] = (b << 32) | (0xFFFFFFFFu - len);
    cid[c] = c;
  }
}

// one warp per block slice, lane l = chunk l of the slice: its source labels column-major (pad = n), its partial
__global__ void block_fill_kernel(uint64_t n_slices, const uint32_t *slice_block, const uint64_t *block_slice_first,
                                  const uint64_t *block_chunk_first, const uint64_t *colbase, const uint64_t *sorted_id,
                                  const uint64_t *cbegin, const uint32_t *clen, const uint32_t *crow,
                                  const uint64_t *bkey, const uint64_t *block_ptr, const uint64_t *chunk_of,
                                  const uint64_t *seg_first, uint32_t pad, uint32_t *idx, uint64_t *slot) {
  const int lane = threadIdx.x & 31;
  const uint64_t warps_total = static_cast<uint64_t>(gridDim.x) * (blockDim.x >> 5);
  for (uint64_t s = static_cast<uint64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); s < n_slices;
       s += warps_total) {
    const uint32_t b = slice_block[s];
    const uint64_t p = block_chunk_first[b] + (s - block_slice_first[b]) * kSliceRows + lane;
    uint64_t begin = 0, d = ~0ull;
    uint32_t len = 0;
    if (p < block_chunk_first[b + 1]) {
      const uint64_t c = sorted_id[p];
      const uint64_t r = crow[c];
      begin = cbegin[c];
      len = clen[c];
      d = seg_first[r + 1] - (chunk_of[block_ptr[r + 1]] - c);  // the row's partials end with its block chunks
    }
    const uint64_t c0 = colbase[s];
    const uint32_t width = static_cast<uint32_t>(colbase[s + 1] - c0);
    uint32_t *dst = idx + c0 * kSliceRows + lane;
    for (uint32_t k = 0; k < width; ++k)
      dst[static_cast<size_t>(k) * kSliceRows] = k < len ? static_cast<uint32_t>(bkey[begin + k]) : pad;
    slot[s * kSliceRows + lane] = d;
  }
}

// ---- SELL staging ----------------------------------------------------------------------------------------------

// Key of SELL entry i: (launch index of its source's block << kStagePosBits) | i when the source lies in a block that
// has a pass, else ~0 (the entry keeps its label: sources below block_from, the pad slot n, blocks without a pass)
constexpr int kStagePosBits = 40;
struct StageKey {
  const uint32_t *idx;       // sell_idx, plain labels
  const uint32_t *launched;  // [blocks] launch index of every label block, ~0 = no pass
  uint64_t from, labels, n;
  __device__ uint64_t operator()(uint64_t i) const {
    const uint32_t l = idx[i];
    if (l < from || l >= n) return ~0ull;
    const uint32_t j = launched[(l - from) / labels];
    return j == ~0u ? ~0ull : (static_cast<uint64_t>(j) << kStagePosBits) | i;
  }
};
struct IsStaged {  // predicate and 0/1 count of a StageKey
  __device__ uint64_t operator()(uint64_t key) const { return key != ~0ull; }
};

// slot q = rank of its key in (block, position) order: stage_src[q] = the entry's label, the entry becomes the slot
__global__ void stage_fill_kernel(uint64_t count, const uint64_t *key, uint32_t *sell_idx, uint32_t *stage_src) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t q = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; q < count; q += stride) {
    const uint64_t i = key[q] & ((1ull << kStagePosBits) - 1);
    stage_src[q] = sell_idx[i];
    sell_idx[i] = kIdxStaged | static_cast<uint32_t>(q);
  }
}

// first[j] = first slot of launched block j (j <= blocks: first[blocks] = count)
__global__ void stage_first_kernel(uint32_t blocks, uint64_t count, const uint64_t *key, uint64_t *first) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j <= blocks) first[j] = lower_bound_key(key, 0, count, static_cast<uint64_t>(j) << kStagePosBits);
}

// work items for the streaming SELL kernel: item i starts at the first slice whose column base is
// >= i * total_cols / n_items (binary search over the slice column bases)
__global__ void sell_items_kernel(uint32_t n_items, uint64_t n_slices, const uint64_t *colbase, uint64_t total_cols,
                                  uint64_t slice_cost, uint64_t *item_begin) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_items) return;
  if (i == n_items) {
    item_begin[i] = n_slices;
    return;
  }
  // cost of slices [0, s) = their columns + slice_cost per slice; item i starts where that reaches i/n_items of the total
  const unsigned __int128 t = static_cast<unsigned __int128>(total_cols + slice_cost * n_slices) * i;
  const uint64_t target = static_cast<uint64_t>(t / n_items);
  uint64_t lo = 0, hi = n_slices;  // first s in [0, n_slices] with cost(s) >= target
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (colbase[mid] + slice_cost * mid < target) lo = mid + 1; else hi = mid;
  }
  item_begin[i] = lo;
}

__global__ void work_item_kernel(uint32_t n_items, const uint64_t *item_begin, const uint64_t *colbase, WorkItem *out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items) return;
  const uint64_t b = item_begin[i], e = item_begin[i + 1];
  WorkItem w{b, e, 0, 0};
  if (b < e) {
    w.col_begin = colbase[b];
    w.col_end = colbase[e];
  }
  out[i] = w;
}

// by_local[r] = by_label[label of this partition's local row r]  (original vertex ids, in-degrees)
__global__ void gather_local_u32_kernel(uint64_t rows, RowMap map, const uint32_t *by_label, uint32_t *by_local) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t r = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < rows; r += stride)
    by_local[r] = by_label[map.label_of_local(r)];
}

__global__ void narrow_kernel(uint64_t count, uint64_t n, const uint64_t *in, uint32_t *out, int *bad) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t e = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < count; e += stride) {
    const uint64_t v = in[e];
    if (v >= n) *bad = 1;
    out[e] = static_cast<uint32_t>(v);
  }
}

// CUB's two-phase call: the first call sizes the scratch, which is taken from `tmp`; the second does the work
template <typename Call>
cudaError_t cub_call(DeviceBuffers &tmp, Call call) {
  size_t bytes = 0;
  cudaError_t e = call(nullptr, bytes);
  if (e != cudaSuccess) return e;
  char *scratch = nullptr;
  if ((e = tmp.alloc(&scratch, bytes)) != cudaSuccess) return e;
  return call(scratch, bytes);
}

// out[0] = 0, out[i + 1] = in[0] + .. + in[i]: an exclusive scan that ends with the total
template <typename It>
cudaError_t prefix_sum(DeviceBuffers &tmp, It in, uint64_t *out, uint64_t count, cudaStream_t st) {
  const cudaError_t e = cudaMemsetAsync(out, 0, sizeof(uint64_t), st);
  if (e != cudaSuccess || count == 0) return e;
  return cub_call(tmp, [&](void *t, size_t &bytes) { return cub::DeviceScan::InclusiveSum(t, bytes, in, out + 1, count, st); });
}

// A device array the graph keeps: counted in resident_bytes and recorded for free_graph
template <typename T>
cudaError_t keep_alloc(Graph &g, T **out, uint64_t count) {
  void *p = nullptr;
  const uint64_t bytes = std::max<uint64_t>(count, 1) * sizeof(T);
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e == cudaSuccess) {
    g.resident_bytes += bytes;
    g.device_arrays.push_back(p);
  }
  *out = static_cast<T *>(p);
  return e;
}

// peak device memory in use during the build (whole device, so other handles of the process count too)
void note_mem(Graph &g) {
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) g.build_peak_bytes = std::max<uint64_t>(g.build_peak_bytes, total_b - free_b);
}

uint32_t env_u32(const char *name, uint32_t fallback) {
  const char *s = getenv(name);
  if (!s || !*s) return fallback;
  const unsigned long v = strtoul(s, nullptr, 10);
  return v ? static_cast<uint32_t>(v) : fallback;
}

uint32_t env_u32_zero(const char *name, uint32_t fallback) {  // like env_u32, but "0" is a value
  const char *s = getenv(name);
  return (s && *s) ? static_cast<uint32_t>(strtoul(s, nullptr, 10)) : fallback;
}

int bits_for(uint64_t v) {  // number of bits needed to represent values < v
  int b = 0;
  while (b < 64 && (v >> b) != 0) ++b;
  return std::max(b, 1);
}

int open_streams(Graph &g) {
  MGB_CUDA(cudaStreamCreateWithFlags(&g.stream, cudaStreamNonBlocking));
  // the side stream carries the SELL epilogue + peer push: highest priority, so that its few CTAs are placed before
  // the heavy-row kernel's when both become ready at the end of the SELL kernel
  int prio_low = 0, prio_high = 0;
  MGB_CUDA(cudaDeviceGetStreamPriorityRange(&prio_low, &prio_high));
  MGB_CUDA(cudaStreamCreateWithPriority(&g.stream2, cudaStreamNonBlocking, prio_high));
  MGB_CUDA(cudaEventCreateWithFlags(&g.fork_ev, cudaEventDisableTiming));
  MGB_CUDA(cudaEventCreateWithFlags(&g.join_ev, cudaEventDisableTiming));
  MGB_CUDA(cudaStreamCreateWithFlags(&g.cold_stream, cudaStreamNonBlocking));
  MGB_CUDA(cudaEventCreateWithFlags(&g.cold_fork_ev, cudaEventDisableTiming));
  MGB_CUDA(cudaEventCreateWithFlags(&g.cold_join_ev, cudaEventDisableTiming));
  return MGB200_OK;
}

// Graph::tun from the environment (g.sm_count sets the defaults of the per-SM counts)
void read_tunables(Graph &g, bool weighted) {
  Graph::Tunables &t = g.tun;
  const char *s = getenv("MGB200_OVERLAP_EPILOGUE");
  g.overlap_epilogue = !(s && s[0] == '0');
  if ((s = getenv("MGB200_L2_HOT_MB")) != nullptr) t.l2_hot_mb = static_cast<uint64_t>(std::max(0l, strtol(s, nullptr, 10)));
  if ((s = getenv("MGB200_L1_HOT_K")) != nullptr) t.l1_hot_k = strtol(s, nullptr, 10);
  if ((s = getenv("MGB200_MULTI_AWARE")) != nullptr) t.multi_aware = s[0] != '0';
  if ((s = getenv("MGB200_FORCE_MULTI_PATH")) != nullptr) t.force_multi_path = s[0] == '1';
  if ((s = getenv("MGB200_SELL_KERNEL")) != nullptr) t.stream_kernel = strcmp(s, "stream") == 0;
  if ((s = getenv("MGB200_IDX_FLAGS")) != nullptr) t.idx_flags = atoi(s);
  if ((s = getenv("MGB200_SELL_MODE")) != nullptr) t.sell_mode = atoi(s);
  if ((s = getenv("MGB200_PUSH_CTAS")) != nullptr) t.push_ctas = std::max(0, atoi(s));
  if ((s = getenv("MGB200_SMEM_TABLE_KB")) != nullptr) t.smem_table_kb = std::max(0l, strtol(s, nullptr, 10));
  if ((s = getenv("MGB200_LABELLING")) != nullptr) t.global_order = strcmp(s, "global") == 0;
  if ((s = getenv("MGB200_PUSH_MASK")) != nullptr) t.push_mask = s[0] == '1';
  if ((s = getenv("MGB200_LONE_PARTITION")) != nullptr) t.lone_partition = s[0] == '1';
  if ((s = getenv("MGB200_TILE_LABELS")) != nullptr)
    t.tile_labels = static_cast<uint32_t>(std::min<unsigned long>(kMaxTileLabels, strtoul(s, nullptr, 10))) & ~1u;
  if ((s = getenv("MGB200_TILE_HOT_MB")) != nullptr) t.tile_hot_mb = std::min<uint64_t>(1ull << 20, strtoull(s, nullptr, 10));
  t.tile_chunk = env_u32("MGB200_TILE_CHUNK", t.tile_chunk);
  if ((s = getenv("MGB200_BLOCK_FROM")) != nullptr) t.block_from = std::min<uint64_t>(strtoull(s, nullptr, 10), ~0u);
  if ((s = getenv("MGB200_BLOCK_LABELS")) != nullptr) t.block_labels = strtoull(s, nullptr, 10);
  t.block_chunk = env_u32("MGB200_BLOCK_CHUNK", t.block_chunk);
  if ((s = getenv("MGB200_SELL_STAGE")) != nullptr) t.sell_stage = s[0] == '1' ? 1 : 0;
  if ((s = getenv("MGB200_BARRIER_TIMEOUT_MS")) != nullptr) {
    const unsigned long long ms = strtoull(s, nullptr, 10);
    if (ms) t.barrier_timeout_ms = ms;
  }
  t.heavy_min_degree = env_u32("MGB200_HEAVY_MIN_DEGREE", t.heavy_min_degree);
  if (getenv("MGB200_SEGMENT_EDGES")) t.segment_edges = env_u32("MGB200_SEGMENT_EDGES", 4096);
  t.tile_runs = env_u32("MGB200_TILE_RUNS", static_cast<uint32_t>(g.sm_count) * 8u);
  t.sell_items = env_u32("MGB200_SELL_ITEMS", static_cast<uint32_t>(g.sm_count) * 32u);
  t.slice_cost = env_u32_zero("MGB200_SLICE_COST", t.slice_cost);
  t.sell_work_items = env_u32("MGB200_SELL_WORK_ITEMS", 0);
  if (weighted) {  // weighted gathers exist on the range path only: the knobs that leave it do not apply
    t.idx_flags = 0;
    t.force_multi_path = false;
  }
}

// What the steps of one build hand each other.  Every device transient comes from `tmp`, the build's one scratch
// arena, and lives until build_graph returns.
struct Build {
  EdgeSource &edges;
  bool weighted;
  uint64_t l2_bytes;  // the device's L2 (sell_staging's default)
  Dealer deal;
  DeviceBuffers tmp;
  IndexFlags heavy_flags{}, sell_flags{};  // stored-index flags of the heavy rows' cold edges and of the SELL entries
  uint64_t chunk_cap = 0;                  // edges per EdgeSource::get()
  uint64_t nonzero_global = 0;             // rows with in-edges in the whole graph (global-order labelling)
  uint32_t *indeg_l = nullptr;             // [n] in-degree by label
  const uint32_t *indeg_local = nullptr;   // [local_rows] in-degree of every owned row
  unsigned long long *counts = nullptr;    // [4] heavy rows, rows with in-edges, edges; owned-edge cursor
  uint64_t *ekey = nullptr, *ekey_alt = nullptr;  // [local_edges] (local row, source label) keys, sorted; spare buffer
  double *eval = nullptr;                  // [local_edges] the edge weights in key order (weighted graphs)
  uint64_t *row_ptr = nullptr;             // [local_rows + 1]
  bool block_on = false;                   // block class: block_edges -> heavy_class, block_slices, sell_staging
  uint64_t block_from = 0, block_labels = 0;
  uint64_t *block_ptr = nullptr, *bkey = nullptr, *bstart = nullptr, *chunk_of = nullptr;
  std::vector<uint32_t> launched_of;       // [blocks] launch index of every label block, ~0 = empty (no pass)
  uint32_t tile_labels = 0;                // tile class: heavy_class -> tile_slices
  uint32_t *tile_lo = nullptr, *pair_cnt = nullptr;
  uint64_t *pair_chunk_first = nullptr;
  unsigned long long *tile_chunks = nullptr;  // [n_tiles] chunks per tile
};

void map_rows(Graph &g, Build &b) {
  RowMap &map = g.map;
  map = RowMap{};
  map.n = g.n;
  map.world = g.part_world;
  map.rank = g.part_rank;
  map.global_order = (g.tun.global_order && g.part_world > 1) ? 1u : 0u;  // one partition: both labellings coincide
  // Hot flags in the stored indices replace the per-gather owner lookup on several partitions (default there);
  // on one partition the range policy already costs nothing per gather, so flags are opt-in (MGB200_IDX_FLAGS=1).
  // They need two index bits (n < 2^30) and partition-aware thresholds; the TMA stream kernel reads raw indices.
  g.idx_flagged = (g.tun.idx_flags > 0 || (g.tun.idx_flags < 0 && g.part_world > 1)) && g.tun.multi_aware &&
                  !g.tun.global_order && !g.tun.stream_kernel && g.n < (1ull << 30);
  // (table_labels() needs idx_flagged, set just above; the heavy-row kernel has no table, so its indices keep labels)
  b.heavy_flags = IndexFlags{b.deal, g.l1_hot_labels(), g.l2_hot_labels(), g.idx_flagged ? 1u : 0u, 0u};
  b.sell_flags = IndexFlags{b.deal, g.l1_hot_labels(), g.l2_hot_labels(), g.idx_flagged ? 1u : 0u,
                            g.idx_flagged ? g.table_labels() / g.part_world : 0u};
  g.row_lo = 0;
  g.local_rows = 0;  // known once the degrees are (global order: depends on the heavy-row count of the whole graph)
}

// iteration state and exchange window exist even for an empty graph
int iteration_state(Graph &g) {
  const cudaStream_t st = g.stream;
  MGB_CUDA(keep_alloc(g, &g.state, 1));
  MGB_CUDA(cudaMemsetAsync(g.state, 0, sizeof(IterState), st));
  MGB_CUDA(cudaMallocHost(reinterpret_cast<void **>(&g.host_state), sizeof(IterState)));
  MGB_CUDA(keep_alloc(g, &g.sum_partials, kSumBlocks));
  MGB_CUDA(keep_alloc(g, &g.queue, 1));
  MGB_CUDA(cudaMemsetAsync(g.queue, 0, sizeof(WorkQueue), st));
  MGB_CUDA(keep_alloc(g, &g.tile_queue, 1));
  MGB_CUDA(cudaMemsetAsync(g.tile_queue, 0, sizeof(WorkQueue), st));
  g.contrib_stride = ((g.n + 1) * sizeof(double) + 255) / 256 * 256;
  g.window_bytes = kFlagPageBytes + 2 * g.contrib_stride;
  MGB_CUDA(keep_alloc(g, reinterpret_cast<char **>(&g.window), g.window_bytes));
  MGB_CUDA(cudaMemsetAsync(g.window, 0, g.window_bytes, st));
  for (int q = 0; q < kMaxPeers; ++q) {
    g.peers.contrib[0][q] = g.peers.contrib[1][q] = nullptr;
    g.peers.flags[q] = nullptr;
  }
  g.peers.contrib[0][g.part_rank] = g.contrib(0);
  g.peers.contrib[1][g.part_rank] = g.contrib(1);
  g.peers.flags[g.part_rank] = g.flags();
  MGB_CUDA(keep_alloc(g, &g.label_of, g.n));
  MGB_CUDA(keep_alloc(g, &g.outdeg_l, g.n));
  return MGB200_OK;
}

int labels(Graph &g, Build &b) {
  RowMap &map = g.map;
  const cudaStream_t st = g.stream;
  const uint64_t n = g.n, m = g.m;
  // 1. degrees in original id space
  uint32_t *outdeg = nullptr, *indeg = nullptr;
  int *bad = nullptr;
  MGB_CUDA(b.tmp.alloc(&outdeg, n));
  MGB_CUDA(b.tmp.alloc(&indeg, n));
  MGB_CUDA(b.tmp.alloc(&bad, 1));
  MGB_CUDA(cudaMemsetAsync(outdeg, 0, n * sizeof(uint32_t), st));
  MGB_CUDA(cudaMemsetAsync(indeg, 0, n * sizeof(uint32_t), st));
  MGB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), st));
  b.chunk_cap = std::max<uint64_t>(1, std::min<uint64_t>(b.edges.chunk_edges ? b.edges.chunk_edges : m, std::max<uint64_t>(m, 1)));
  for (uint64_t first = 0; first < m; first += b.chunk_cap) {  // pass 1 over the edge list: degrees
    const uint64_t cnt = std::min(b.chunk_cap, m - first);
    const uint32_t *d_from = nullptr, *d_to = nullptr;
    const int grc = b.edges.get(first, cnt, &d_from, &d_to, st);
    if (grc) return grc;
    degree_kernel<<<blocks_for(cnt, g.sm_count, 16), kThreads, 0, st>>>(cnt, n, d_from, d_to, outdeg, indeg, bad);
  }
  int bad_host = 0;
  MGB_CUDA(cudaMemcpyAsync(&bad_host, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  if (bad_host) {
    set_error("edge endpoint out of range (>= number_of_nodes)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }

  // 1b. who owns what.  Global-order labelling deals the heavy rows singly and the rest in blocks of 32 labels, so it
  // needs the heavy-row count (and, for the zero-row tail, the non-zero count) of the WHOLE graph first.
  if (map.global_order) {
    unsigned long long *gc = nullptr;
    MGB_CUDA(b.tmp.alloc(&gc, 3));
    MGB_CUDA(cudaMemsetAsync(gc, 0, 3 * sizeof(unsigned long long), st));
    class_count_kernel<<<blocks_for(n, g.sm_count, 16), kThreads, 0, st>>>(n, indeg, g.tun.heavy_min_degree, gc);
    unsigned long long gc_host[3] = {0, 0, 0};
    MGB_CUDA(cudaMemcpyAsync(gc_host, gc, sizeof(gc_host), cudaMemcpyDeviceToHost, st));
    MGB_CUDA(cudaStreamSynchronize(st));
    map.heavy = gc_host[0];
    b.nonzero_global = std::max<uint64_t>(gc_host[1], gc_host[0]);
  }
  map.finalize();
  g.row_lo = map.row_lo;
  g.local_rows = map.local_rows(g.part_rank);
  MGB_CUDA(keep_alloc(g, &g.rank, g.local_rows));
  MGB_CUDA(keep_alloc(g, &g.local_vertex, g.local_rows));

  // 2. global order: in-degree desc, out-degree desc, id asc (stable radix sort)
  uint64_t *vkey = nullptr, *vkey_alt = nullptr;
  uint32_t *vid = nullptr, *vid_alt = nullptr;
  MGB_CUDA(b.tmp.alloc(&vkey, n));
  MGB_CUDA(b.tmp.alloc(&vkey_alt, n));
  MGB_CUDA(b.tmp.alloc(&vid, n));
  MGB_CUDA(b.tmp.alloc(&vid_alt, n));
  sort_key_kernel<<<blocks_for(n, g.sm_count, 16), kThreads, 0, st>>>(n, indeg, outdeg, vkey, vid);
  cub::DoubleBuffer<uint64_t> kb(vkey, vkey_alt);
  cub::DoubleBuffer<uint32_t> vb(vid, vid_alt);
  MGB_CUDA(cub_call(b.tmp, [&](void *t, size_t &bytes) { return cub::DeviceRadixSort::SortPairs(t, bytes, kb, vb, n, 0, 64, st); }));
  vid = vb.Current();

  // 3. labels, degrees by label
  uint32_t *vertex_of_label = nullptr;
  MGB_CUDA(b.tmp.alloc(&b.indeg_l, n));
  MGB_CUDA(b.tmp.alloc(&vertex_of_label, n));
  label_kernel<<<blocks_for(n, g.sm_count, 16), kThreads, 0, st>>>(map, vid, indeg, outdeg, g.label_of, b.indeg_l,
                                                              g.outdeg_l, vertex_of_label);
  gather_local_u32_kernel<<<blocks_for(g.local_rows, g.sm_count, 16), kThreads, 0, st>>>(g.local_rows, map, vertex_of_label,
                                                                                    g.local_vertex);
  b.indeg_local = b.indeg_l + g.row_lo;  // dealt ranges: the owned labels are contiguous
  if (map.global_order) {
    uint32_t *gathered = nullptr;
    MGB_CUDA(b.tmp.alloc(&gathered, g.local_rows));
    gather_local_u32_kernel<<<blocks_for(g.local_rows, g.sm_count, 16), kThreads, 0, st>>>(g.local_rows, map, b.indeg_l,
                                                                                      gathered);
    b.indeg_local = gathered;
  }
  if (g.tun.push_mask && g.part_world > 1 && m > 0 && g.local_rows > 0) {
    const uint64_t words = (g.local_rows + 3) / 4;
    MGB_CUDA(keep_alloc(g, &g.need_mask, words));
    MGB_CUDA(cudaMemsetAsync(g.need_mask, 0, words * sizeof(uint32_t), st));
    // filled in pass 2 over the edge list, next to the owned-edge extraction
  }
  return MGB200_OK;
}

// 4. class boundaries and local edge count
int row_classes(Graph &g, Build &b) {
  const RowMap &map = g.map;
  const cudaStream_t st = g.stream;
  const uint64_t n = g.n;
  MGB_CUDA(b.tmp.alloc(&b.counts, 4));
  MGB_CUDA(cudaMemsetAsync(b.counts, 0, 4 * sizeof(unsigned long long), st));
  class_count_kernel<<<blocks_for(g.local_rows, g.sm_count, 16), kThreads, 0, st>>>(g.local_rows, b.indeg_local,
                                                                               g.tun.heavy_min_degree, b.counts);
  unsigned long long counts_host[4] = {0, 0, 0, 0};
  MGB_CUDA(cudaMemcpyAsync(counts_host, b.counts, sizeof(counts_host), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  g.any_zero_rows = false;
  uint64_t sell_rows_global_order = 0;
  if (map.global_order) {
    // Blocks [0, nz_blocks) hold at least one row with in-edges: they are SELL slices (the zero rows of the one mixed
    // block are ordinary SELL rows of width 0).  Every label from zero_first on is a zero row on whichever partition
    // owns it: ONE global tail range, the same on every partition.
    const uint64_t nz_blocks =
        b.nonzero_global > map.heavy ? (b.nonzero_global - map.heavy + kSliceRows - 1) / kSliceRows : 0;
    const uint64_t zero_first = std::min<uint64_t>(n, map.heavy + nz_blocks * kSliceRows);
    sell_rows_global_order = map.rows_in_blocks(g.part_rank, nz_blocks);
    for (uint32_t q = 0; q < g.part_world; ++q) g.part_start[q] = g.zero_lo[q] = g.zero_hi[q] = 0;
    g.zero_lo[0] = zero_first;
    g.zero_hi[0] = n;
    g.any_zero_rows = zero_first < n;
  } else {
    unsigned long long *nz = nullptr;
    MGB_CUDA(b.tmp.alloc(&nz, kMaxPeers));
    MGB_CUDA(cudaMemsetAsync(nz, 0, kMaxPeers * sizeof(unsigned long long), st));
    nonzero_per_partition_kernel<<<blocks_for(n / g.part_world + 1, g.sm_count, 16), kThreads, 0, st>>>(b.deal, b.indeg_l, nz);
    unsigned long long nz_host[kMaxPeers] = {};
    MGB_CUDA(cudaMemcpyAsync(nz_host, nz, sizeof(nz_host), cudaMemcpyDeviceToHost, st));
    MGB_CUDA(cudaStreamSynchronize(st));
    for (uint32_t q = 0; q < g.part_world; ++q) {
      g.part_start[q] = b.deal.start(q);
      g.zero_lo[q] = b.deal.start(q) + nz_host[q];
      g.zero_hi[q] = b.deal.start(q) + b.deal.count(q);
      if (g.zero_hi[q] > g.zero_lo[q]) g.any_zero_rows = true;
    }
  }
  g.n_heavy = counts_host[0];
  if (map.global_order && g.n_heavy != map.heavy_q) {
    set_error("internal: heavy rows owned (" + std::to_string(g.n_heavy) + ") != dealt (" + std::to_string(map.heavy_q) + ")");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  g.n_sell = map.global_order ? sell_rows_global_order : counts_host[1] - counts_host[0];
  g.n_zero = g.local_rows - g.n_heavy - g.n_sell;
  g.local_edges = counts_host[2];
  return MGB200_OK;
}

// 5. keys of the owned edges, sorted by (local row, source label)
int edge_keys(Graph &g, Build &b) {
  const cudaStream_t st = g.stream;
  const uint64_t n = g.n, m = g.m;
  MGB_CUDA(b.tmp.alloc(&b.ekey, g.local_edges));
  MGB_CUDA(b.tmp.alloc(&b.ekey_alt, g.local_edges));
  if (b.weighted && g.part_world > 1) {
    set_error("edge weights are supported on a single partition only");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  double *eval_alt = nullptr;  // b.eval: weights travelling with the edge keys through the sort
  if (b.weighted) {
    MGB_CUDA(b.tmp.alloc(&b.eval, g.local_edges));
    MGB_CUDA(b.tmp.alloc(&eval_alt, g.local_edges));
    MGB_CUDA(keep_alloc(g, &g.outw_l, n));
    MGB_CUDA(cudaMemsetAsync(g.outw_l, 0, n * sizeof(double), st));
  }
  if (m && g.part_world > 1) MGB_CUDA(cudaMemsetAsync(b.counts + 3, 0, sizeof(unsigned long long), st));
  const uint64_t row_hi = g.row_lo + g.local_rows;
  for (uint64_t first = 0; first < m; first += b.chunk_cap) {  // pass 2 over the edge list: who reads what, owned edges
    const uint64_t cnt = std::min(b.chunk_cap, m - first);
    const uint32_t *d_from = nullptr, *d_to = nullptr;
    const int grc = b.edges.get(first, cnt, &d_from, &d_to, st);
    if (grc) return grc;
    if (g.need_mask)
      need_mask_kernel<<<blocks_for(cnt, g.sm_count, 16), kThreads, 0, st>>>(cnt, d_from, d_to, g.label_of, g.map, g.need_mask);
    if (g.part_world == 1) {
      edge_key_all_kernel<<<blocks_for(cnt, g.sm_count, 16), kThreads, 0, st>>>(cnt, d_from, d_to, g.label_of, b.ekey + first);
      if (b.weighted) {
        const double *d_w = b.edges.weights();
        MGB_CUDA(cudaMemcpyAsync(b.eval + first, d_w, cnt * sizeof(double), cudaMemcpyDeviceToDevice, st));
        out_weight_kernel<<<blocks_for(cnt, g.sm_count, 16), kThreads, 0, st>>>(cnt, d_from, d_w, g.label_of, g.outw_l);
      }
    } else {
      edge_key_owned_kernel<<<blocks_for(cnt, g.sm_count, 16), kThreads, 0, st>>>(cnt, d_from, d_to, g.label_of, g.map,
                                                                             row_hi, b.ekey, b.counts + 3);
    }
  }
  note_mem(g);
  if (g.local_edges) {
    cub::DoubleBuffer<uint64_t> kb(b.ekey, b.ekey_alt);
    const int end_bit = std::min(64, 32 + bits_for(g.local_rows));
    if (b.weighted) {
      cub::DoubleBuffer<double> vb(b.eval, eval_alt);
      MGB_CUDA(cub_call(b.tmp, [&](void *t, size_t &bytes) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, kb, vb, g.local_edges, 0, end_bit, st);
      }));
      b.eval = vb.Current();
    } else {
      MGB_CUDA(cub_call(b.tmp, [&](void *t, size_t &bytes) {
        return cub::DeviceRadixSort::SortKeys(t, bytes, kb, g.local_edges, 0, end_bit, st);
      }));
    }
    note_mem(g);
    b.ekey = kb.Current();
    b.ekey_alt = kb.Alternate();  // free again: the heavy rows' cold keys are compacted into it
  }
  return MGB200_OK;
}

// 6. row pointers over the local rows (uint64)
int row_pointers(Graph &g, Build &b) {
  MGB_CUDA(b.tmp.alloc(&b.row_ptr, g.local_rows + 1));
  cub::TransformInputIterator<uint64_t, U32ToU64, const uint32_t *> it(b.indeg_local, U32ToU64());
  MGB_CUDA(prefix_sum(b.tmp, it, b.row_ptr, g.local_rows, g.stream));
  return MGB200_OK;
}

// 6b. block class (one partition, unweighted, labels past block_from): the heavy rows' sources >= block_from are
// gathered one L2-sized label block at a time (block_slices).  Heavy rows come first in key order, so their keys are
// the first heavy-edge keys; those >= block_from are compacted (row-major, ascending sources) and cut into chunks of at
// most block_chunk edges of one (row, block) run.
int block_edges(Graph &g, Build &b) {
  const cudaStream_t st = g.stream;
  const uint64_t n = g.n;
  b.block_from = g.tun.block_from;
  b.block_on = g.part_world == 1 && !g.tun.force_multi_path && !b.weighted && g.tun.block_labels > 0 &&
               n > b.block_from && n < (1ull << 32) - 1;
  // at most kMaxBlocks launches per gather: a smaller MGB200_BLOCK_LABELS is raised to that
  b.block_labels =
      b.block_on ? std::max<uint64_t>(g.tun.block_labels, (n - b.block_from + kMaxBlocks - 1) / kMaxBlocks) : 0;
  g.block_labels = b.block_labels;
  if (!b.block_on || !g.n_heavy) return MGB200_OK;
  const uint64_t nh = g.n_heavy;
  uint64_t *block_cnt = nullptr, heavy_edges = 0;
  MGB_CUDA(b.tmp.alloc(&block_cnt, nh));
  MGB_CUDA(b.tmp.alloc(&b.block_ptr, nh + 1));
  block_row_kernel<<<blocks_for(nh, g.sm_count, 16), kThreads, 0, st>>>(nh, b.row_ptr, b.ekey, b.block_from, block_cnt);
  MGB_CUDA(prefix_sum(b.tmp, block_cnt, b.block_ptr, nh, st));
  MGB_CUDA(cudaMemcpyAsync(&g.block_edges, b.block_ptr + nh, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaMemcpyAsync(&heavy_edges, b.row_ptr + nh, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  if (!g.block_edges) return MGB200_OK;
  const uint64_t ne = g.block_edges;
  MGB_CUDA(b.tmp.alloc(&b.bkey, ne));
  MGB_CUDA(b.tmp.alloc(&b.bstart, ne));
  MGB_CUDA(b.tmp.alloc(&b.chunk_of, ne + 1));
  unsigned long long *d_sel = nullptr;
  MGB_CUDA(b.tmp.alloc(&d_sel, 1));
  MGB_CUDA(cub_call(b.tmp, [&](void *t, size_t &bytes) {
    return cub::DeviceSelect::If(t, bytes, b.ekey, b.bkey, d_sel, static_cast<int64_t>(heavy_edges), BlockKey{b.block_from}, st);
  }));
  block_start_kernel<<<blocks_for(ne, g.sm_count, 16), kThreads, 0, st>>>(ne, b.bkey, b.block_ptr, b.block_from,
                                                                      b.block_labels, g.tun.block_chunk, b.bstart);
  MGB_CUDA(prefix_sum(b.tmp, b.bstart, b.chunk_of, ne, st));  // chunk_of[i] = chunk of a starting edge i
  MGB_CUDA(cudaMemcpyAsync(&g.block_chunks, b.chunk_of + ne, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  note_mem(g);
  return MGB200_OK;
}

// 7. heavy class: tile chunks of the hot sources (tile_slices), CSC + segments of the cold ones, block chunks of the
// rest (block_slices)
int heavy_class(Graph &g, Build &b) {
  const cudaStream_t st = g.stream;
  const uint64_t n = g.n, nh = g.n_heavy;
  MGB_CUDA(cudaMemcpyAsync(&g.heavy_edges, b.row_ptr + nh, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  // 7a. tiles: every owner's hot prefix cut into T-label windows; a window starts on an even label (16-byte aligned)
  const uint32_t T = b.tile_labels = b.weighted ? 0u : g.tun.tile_labels;
  const uint32_t owners = (g.part_world > 1 && !g.map.global_order) ? g.part_world : 1u;
  uint64_t tile_hot = T ? (g.tun.tile_hot_mb << 20) / sizeof(double) / owners : 0;
  if (b.block_on) tile_hot = std::min(tile_hot, b.block_from);  // sources past block_from belong to the block class
  const TileSet tiles{Dealer{n, owners}, tile_hot};
  std::vector<uint32_t> t_lo, t_hi, t_base, t_load;
  for (uint32_t q = 0; T && q < owners; ++q) {
    const uint64_t s0 = tiles.owners.start(q), end = s0 + std::min(tiles.hot, tiles.owners.count(q));
    for (uint64_t t = s0 & ~1ull; t < end; t += T) {
      t_lo.push_back(static_cast<uint32_t>(std::max(t, s0)));
      t_hi.push_back(static_cast<uint32_t>(std::min(t + T, end)));
      t_base.push_back(static_cast<uint32_t>(t));
      t_load.push_back(static_cast<uint32_t>((std::min(t + T, end) - t + 1) & ~1ull));
    }
  }
  const uint32_t nt = static_cast<uint32_t>(t_lo.size());
  g.n_tiles = nt;
  const uint64_t pairs = nh * nt;
  uint32_t *d_hi = nullptr;
  uint64_t *pair_chunks = nullptr;
  if (nt) {
    MGB_CUDA(b.tmp.alloc(&b.tile_lo, nt));
    MGB_CUDA(b.tmp.alloc(&d_hi, nt));
    MGB_CUDA(keep_alloc(g, &g.tile_base, nt));
    MGB_CUDA(keep_alloc(g, &g.tile_load, nt));
    MGB_CUDA(cudaMemcpyAsync(b.tile_lo, t_lo.data(), nt * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    MGB_CUDA(cudaMemcpyAsync(d_hi, t_hi.data(), nt * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    MGB_CUDA(cudaMemcpyAsync(g.tile_base, t_base.data(), nt * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    MGB_CUDA(cudaMemcpyAsync(g.tile_load, t_load.data(), nt * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    MGB_CUDA(b.tmp.alloc(&b.pair_cnt, pairs));
    MGB_CUDA(b.tmp.alloc(&pair_chunks, pairs));
    MGB_CUDA(b.tmp.alloc(&b.pair_chunk_first, pairs + 1));
    MGB_CUDA(b.tmp.alloc(&b.tile_chunks, nt));
    MGB_CUDA(cudaMemsetAsync(b.tile_chunks, 0, nt * sizeof(unsigned long long), st));
    tile_pair_kernel<<<blocks_for(pairs, g.sm_count, 16), kThreads, 0, st>>>(nh, nt, b.row_ptr, b.ekey, b.tile_lo, d_hi,
                                                                          g.tun.tile_chunk, b.pair_cnt, pair_chunks,
                                                                          b.tile_chunks);
    MGB_CUDA(prefix_sum(b.tmp, pair_chunks, b.pair_chunk_first, pairs, st));
  }
  const uint64_t *heavy_block_ptr = g.block_edges ? b.block_ptr : nullptr;  // block edges per heavy row, if any
  uint64_t *cold_deg = nullptr, *row_chunks = nullptr, *row_parts = nullptr, *row_cold_segs = nullptr,
           *cold_seg_first = nullptr;
  MGB_CUDA(b.tmp.alloc(&cold_deg, nh));
  MGB_CUDA(b.tmp.alloc(&row_chunks, nh));
  MGB_CUDA(b.tmp.alloc(&row_parts, nh));
  MGB_CUDA(b.tmp.alloc(&row_cold_segs, nh));
  MGB_CUDA(b.tmp.alloc(&cold_seg_first, nh + 1));
  tile_row_kernel<<<blocks_for(nh, g.sm_count, 16), kThreads, 0, st>>>(nh, nt, b.indeg_local, b.pair_cnt, pair_chunks,
                                                                    heavy_block_ptr, cold_deg, row_chunks);
  MGB_CUDA(keep_alloc(g, &g.heavy_ptr, nh + 1));
  MGB_CUDA(prefix_sum(b.tmp, cold_deg, g.heavy_ptr, nh, st));
  uint64_t cold_edges = 0;
  MGB_CUDA(cudaMemcpyAsync(&cold_edges, g.heavy_ptr + nh, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  if (nt) MGB_CUDA(cudaMemcpyAsync(&g.tile_chunks, b.pair_chunk_first + pairs, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  g.tiled_edges = g.heavy_edges - cold_edges - g.block_edges;
  g.segment_edges = g.tun.segment_edges;
  if (!g.segment_edges) {
    // one warp per segment: aim for >= 8 segments per resident warp (64 warps/SM) so the tail is short
    // when a partition holds few cold heavy edges (multi-GPU, or most of them tiled), capped at 4096 edges
    const uint64_t resident_warps = static_cast<uint64_t>(g.sm_count) * 64;
    uint64_t seg = cold_edges / (resident_warps * 8);
    seg = (seg / 256) * 256;
    g.segment_edges = static_cast<uint32_t>(std::min<uint64_t>(4096, std::max<uint64_t>(256, seg)));
  }
  seg_count_kernel<<<blocks_for(nh, g.sm_count, 16), kThreads, 0, st>>>(nh, cold_deg, row_chunks, heavy_block_ptr,
                                                                     b.chunk_of, g.segment_edges, row_parts, row_cold_segs);
  MGB_CUDA(keep_alloc(g, &g.seg_first, nh + 1));
  MGB_CUDA(prefix_sum(b.tmp, row_parts, g.seg_first, nh, st));
  MGB_CUDA(prefix_sum(b.tmp, row_cold_segs, cold_seg_first, nh, st));
  MGB_CUDA(cudaMemcpyAsync(&g.n_seg, g.seg_first + nh, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaMemcpyAsync(&g.n_cold_seg, cold_seg_first + nh, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  // 7b. cold edges: the heavy rows' keys without the tiled and block ones (order kept), as CSC + fixed-size segments
  const uint64_t *cold_keys = b.ekey;
  if (g.tiled_edges || g.block_edges) {
    unsigned long long *d_sel = nullptr;
    MGB_CUDA(b.tmp.alloc(&d_sel, 1));
    const ColdKey cold{tiles, b.block_on ? b.block_from : n + 1};
    MGB_CUDA(cub_call(b.tmp, [&](void *t, size_t &bytes) {
      return cub::DeviceSelect::If(t, bytes, b.ekey, b.ekey_alt, d_sel, static_cast<int64_t>(g.heavy_edges), cold, st);
    }));
    cold_keys = b.ekey_alt;
  }
  MGB_CUDA(keep_alloc(g, &g.heavy_idx, cold_edges));
  low32_kernel<<<blocks_for(cold_edges, g.sm_count, 16), kThreads, 0, st>>>(cold_edges, cold_keys, b.heavy_flags,
                                                                         g.heavy_idx);
  if (b.weighted) {  // rows are sorted, heavy rows first: their weights are the prefix of the sorted weights (no tiles)
    MGB_CUDA(keep_alloc(g, &g.heavy_w, g.heavy_edges));
    MGB_CUDA(cudaMemcpyAsync(g.heavy_w, b.eval, g.heavy_edges * sizeof(double), cudaMemcpyDeviceToDevice, st));
  }
  MGB_CUDA(cudaStreamSynchronize(st));
  MGB_CUDA(keep_alloc(g, &g.seg_row, g.n_cold_seg));
  MGB_CUDA(keep_alloc(g, &g.seg_begin, g.n_cold_seg));
  if (g.tile_chunks || g.block_chunks) MGB_CUDA(keep_alloc(g, &g.seg_slot, g.n_cold_seg));
  MGB_CUDA(keep_alloc(g, &g.seg_partial, g.n_seg));
  MGB_CUDA(keep_alloc(g, &g.heavy_sums, nh));
  segment_fill_kernel<<<blocks_for(nh * 32, g.sm_count, 16), kThreads, 0, st>>>(
      nh, g.heavy_ptr, cold_seg_first, g.segment_edges, g.seg_first, heavy_block_ptr, b.chunk_of, g.seg_row, g.seg_begin,
      g.seg_slot);
  return MGB200_OK;
}

// Chunks of `groups` groups (tiles or label blocks) -> per group, SELL-32 slices of its chunks sorted by length (ties:
// row order).  In: the chunks per group, and every chunk's (group, length) key, id and length.  The slice tables come
// from the arena, or are kept by the graph with `keep_tables`; the column bases are always kept.
struct ChunkSlices {
  std::vector<uint64_t> slice_first;    // host [groups + 1]: slices are group-major
  uint64_t slices = 0, total_cols = 0;
  uint64_t *chunk_first = nullptr;      // [groups + 1] first chunk of every group, in sorted order
  uint64_t *d_slice_first = nullptr;    // [groups + 1]
  uint32_t *slice_group = nullptr;      // [slices]
  const uint64_t *sorted_id = nullptr;  // [chunks] chunk ids in (group, length) order
  uint64_t *colbase = nullptr;          // [slices + 1] in units of 32-entry columns
};

int slice_chunks(Graph &g, Build &b, uint64_t groups, const unsigned long long *per_group, uint64_t chunks,
                 uint64_t *ckey, uint64_t *cid, const uint32_t *clen, bool keep_tables, ChunkSlices &out) {
  const cudaStream_t st = g.stream;
  std::vector<unsigned long long> counts(groups);
  MGB_CUDA(cudaMemcpyAsync(counts.data(), per_group, groups * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  std::vector<uint64_t> chunk_first(groups + 1, 0);
  std::vector<uint32_t> slice_group;
  out.slice_first.assign(groups + 1, 0);
  for (uint64_t q = 0; q < groups; ++q) {
    chunk_first[q + 1] = chunk_first[q] + counts[q];
    const uint64_t slices = (counts[q] + kSliceRows - 1) / kSliceRows;
    out.slice_first[q + 1] = out.slice_first[q] + slices;
    slice_group.insert(slice_group.end(), slices, static_cast<uint32_t>(q));
  }
  const uint64_t ns = out.slices = out.slice_first[groups];
  MGB_CUDA(b.tmp.alloc(&out.chunk_first, groups + 1));
  MGB_CUDA(keep_tables ? keep_alloc(g, &out.d_slice_first, groups + 1) : b.tmp.alloc(&out.d_slice_first, groups + 1));
  MGB_CUDA(keep_tables ? keep_alloc(g, &out.slice_group, ns) : b.tmp.alloc(&out.slice_group, ns));
  MGB_CUDA(cudaMemcpyAsync(out.chunk_first, chunk_first.data(), (groups + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  MGB_CUDA(cudaMemcpyAsync(out.d_slice_first, out.slice_first.data(), (groups + 1) * sizeof(uint64_t),
                           cudaMemcpyHostToDevice, st));
  MGB_CUDA(cudaMemcpyAsync(out.slice_group, slice_group.data(), ns * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  uint64_t *ckey_alt = nullptr, *cid_alt = nullptr;
  MGB_CUDA(b.tmp.alloc(&ckey_alt, chunks));
  MGB_CUDA(b.tmp.alloc(&cid_alt, chunks));
  cub::DoubleBuffer<uint64_t> kb(ckey, ckey_alt);
  cub::DoubleBuffer<uint64_t> vb(cid, cid_alt);
  const int end_bit = 32 + bits_for(groups);
  // stable: equal (group, length) keep row order, so the layout is a function of the graph alone
  MGB_CUDA(cub_call(b.tmp, [&](void *t, size_t &bytes) {
    return cub::DeviceRadixSort::SortPairs(t, bytes, kb, vb, chunks, 0, end_bit, st);
  }));
  out.sorted_id = vb.Current();
  uint64_t *width = nullptr;
  MGB_CUDA(b.tmp.alloc(&width, ns));
  tile_width_kernel<<<blocks_for(ns, g.sm_count, 16), kThreads, 0, st>>>(ns, out.slice_group, out.d_slice_first,
                                                                      out.chunk_first, out.sorted_id, clen, width);
  MGB_CUDA(keep_alloc(g, &out.colbase, ns + 1));
  MGB_CUDA(prefix_sum(b.tmp, width, out.colbase, ns, st));
  MGB_CUDA(cudaMemcpyAsync(&out.total_cols, out.colbase + ns, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  return MGB200_OK;
}

// 7c. tile chunks -> per tile, SELL-32 slices of chunks sorted by length (ties: row order)
int tile_slices(Graph &g, Build &b) {
  if (!g.tile_chunks) return MGB200_OK;
  const cudaStream_t st = g.stream;
  const uint32_t nt = g.n_tiles;
  const uint64_t nh = g.n_heavy, pairs = nh * nt, nc = g.tile_chunks;
  uint64_t *ckey = nullptr, *cid = nullptr, *cbegin = nullptr, *cslot = nullptr;
  uint32_t *clen = nullptr;
  MGB_CUDA(b.tmp.alloc(&ckey, nc));
  MGB_CUDA(b.tmp.alloc(&cid, nc));
  MGB_CUDA(b.tmp.alloc(&cbegin, nc));
  MGB_CUDA(b.tmp.alloc(&clen, nc));
  MGB_CUDA(b.tmp.alloc(&cslot, nc));
  tile_chunk_kernel<<<blocks_for(pairs, g.sm_count, 16), kThreads, 0, st>>>(nh, nt, b.row_ptr, b.ekey, b.tile_lo,
                                                                       b.pair_cnt, b.pair_chunk_first, g.seg_first,
                                                                       g.tun.tile_chunk, ckey, cid, cbegin, clen, cslot);
  ChunkSlices s;
  if (const int rc = slice_chunks(g, b, nt, b.tile_chunks, nc, ckey, cid, clen, true, s)) return rc;
  const uint64_t ns = g.tile_slices = s.slices;
  g.tile_slice_first = s.d_slice_first;
  g.tslice_tile = s.slice_group;
  g.tslice_colbase = s.colbase;
  MGB_CUDA(keep_alloc(g, &g.tile_idx, s.total_cols * kSliceRows));
  MGB_CUDA(keep_alloc(g, &g.tile_slot, ns * kSliceRows));
  tile_fill_kernel<<<blocks_for(ns * 32, g.sm_count, 16), kThreads, 0, st>>>(
      ns, g.tslice_tile, g.tile_slice_first, s.chunk_first, g.tile_base, g.tslice_colbase, s.sorted_id, cbegin, clen,
      cslot, b.ekey, static_cast<uint16_t>(b.tile_labels), g.tile_idx, g.tile_slot);
  // runs of heavy_tiles_kernel: contiguous slice runs of ~equal cost = columns + 8 per slice, drawn in tile order by
  // one persistent CTA per SM.  8 runs per SM (MGB200_TILE_RUNS sets the total): scale-26 on one H100, one
  // bench.py --quick run each, 4 per SM is slower (8.46 against 8.32 ms per iteration) and 16 is not faster (8.34);
  // a slice cost of 2 is slower (8.41), 24 no faster (8.31), so the SELL items' 8 stays.
  g.tile_work = static_cast<uint32_t>(std::min<uint64_t>(ns, g.tun.tile_runs));
  MGB_CUDA(keep_alloc(g, &g.tile_work_begin, static_cast<uint64_t>(g.tile_work) + 1));
  sell_items_kernel<<<(g.tile_work + 1 + kThreads - 1) / kThreads, kThreads, 0, st>>>(
      g.tile_work, ns, g.tslice_colbase, s.total_cols, 8, g.tile_work_begin);
  return MGB200_OK;
}

// 8. SELL class
int sell_class(Graph &g, Build &b) {
  if (!g.n_sell) return MGB200_OK;
  const cudaStream_t st = g.stream;
  g.n_slices = (g.n_sell + kSliceRows - 1) / kSliceRows;
  uint64_t *width = nullptr;
  MGB_CUDA(b.tmp.alloc(&width, g.n_slices));
  slice_width_kernel<<<blocks_for(g.n_slices, g.sm_count, 16), kThreads, 0, st>>>(g.n_slices, b.indeg_local, g.n_heavy,
                                                                               width);
  MGB_CUDA(keep_alloc(g, &g.sell_colbase, g.n_slices + 1));
  MGB_CUDA(prefix_sum(b.tmp, width, g.sell_colbase, g.n_slices, st));
  uint64_t total_cols = 0;
  MGB_CUDA(cudaMemcpyAsync(&total_cols, g.sell_colbase + g.n_slices, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  g.sell_entries = total_cols * kSliceRows;
  MGB_CUDA(keep_alloc(g, &g.sell_idx, g.sell_entries));
  if (b.weighted) MGB_CUDA(keep_alloc(g, &g.sell_w, g.sell_entries));
  sell_fill_kernel<<<blocks_for(g.n_slices * 32, g.sm_count, 16), kThreads, 0, st>>>(
      g.n_slices, g.n_heavy, g.n_heavy + g.n_sell, b.row_ptr, b.ekey, g.sell_colbase, static_cast<uint32_t>(g.n),
      b.sell_flags, g.sell_idx, b.eval, g.sell_w);
  MGB_CUDA(keep_alloc(g, &g.sell_sums, g.n_sell));
  g.sell_items = g.tun.sell_items;
  MGB_CUDA(keep_alloc(g, &g.sell_item_begin, static_cast<uint64_t>(g.sell_items) + 1));
  sell_items_kernel<<<(g.sell_items + 1 + kThreads - 1) / kThreads, kThreads, 0, st>>>(
      g.sell_items, g.n_slices, g.sell_colbase, total_cols, 0, g.sell_item_begin);
  // Work items of sell_rows_kernel (contiguous slice runs of ~equal cost = columns + slice_cost per slice).
  // With >= 64 slices per resident warp the ticket queue over ~16 items per warp balances best (a whole scale-26
  // graph); below that every extra run start costs more than the balance gains and ONE (or two) contiguous runs per
  // warp, dealt statically, are faster (the partitions of a multi-GPU run).
  // item basis: the warps resident at once in the kernel that will walk them (24 per SM for the plain and the table
  // walk); a deal sized for more warps than run gives some warps one item more than the rest
  const uint64_t resident_warps = static_cast<uint64_t>(g.sm_count) * sell_warps_per_sm(g);
  const uint64_t per_warp = g.n_slices / resident_warps;
  g.sell_static = g.tun.sell_mode >= 0 ? g.tun.sell_mode == 1 : per_warp < 64;
  const uint64_t items_default = !g.sell_static ? resident_warps * 16 : (per_warp < 32 ? resident_warps : resident_warps * 2);
  const uint32_t items = g.tun.sell_work_items ? g.tun.sell_work_items : static_cast<uint32_t>(items_default);
  g.sell_work = static_cast<uint32_t>(std::min<uint64_t>(g.n_slices, items));
  MGB_CUDA(keep_alloc(g, &g.sell_work_begin, static_cast<uint64_t>(g.sell_work) + 1));
  sell_items_kernel<<<(g.sell_work + 1 + kThreads - 1) / kThreads, kThreads, 0, st>>>(
      g.sell_work, g.n_slices, g.sell_colbase, total_cols, g.tun.slice_cost, g.sell_work_begin);
  MGB_CUDA(keep_alloc(g, &g.sell_work_items, g.sell_work));
  work_item_kernel<<<(g.sell_work + kThreads - 1) / kThreads, kThreads, 0, st>>>(g.sell_work, g.sell_work_begin,
                                                                                g.sell_colbase, g.sell_work_items);
  return MGB200_OK;
}

// 9. block chunks -> per block, SELL-32 slices of chunks sorted by length (ties: row order); empty blocks are skipped
int block_slices(Graph &g, Build &b) {
  if (!g.block_chunks) return MGB200_OK;
  const cudaStream_t st = g.stream;
  const uint64_t nb = (g.n - b.block_from + b.block_labels - 1) / b.block_labels, nc = g.block_chunks, ne = g.block_edges;
  uint64_t *cbegin = nullptr, *ckey = nullptr, *cid = nullptr;
  uint32_t *crow = nullptr, *clen = nullptr;
  unsigned long long *per_block = nullptr;
  MGB_CUDA(b.tmp.alloc(&cbegin, nc));
  MGB_CUDA(b.tmp.alloc(&ckey, nc));
  MGB_CUDA(b.tmp.alloc(&cid, nc));
  MGB_CUDA(b.tmp.alloc(&crow, nc));
  MGB_CUDA(b.tmp.alloc(&clen, nc));
  MGB_CUDA(b.tmp.alloc(&per_block, nb));
  MGB_CUDA(cudaMemsetAsync(per_block, 0, nb * sizeof(unsigned long long), st));
  block_chunk_kernel<<<blocks_for(ne, g.sm_count, 16), kThreads, 0, st>>>(ne, b.bkey, b.bstart, b.chunk_of, b.block_from,
                                                                      b.block_labels, cbegin, crow, per_block);
  block_len_kernel<<<blocks_for(nc, g.sm_count, 16), kThreads, 0, st>>>(nc, ne, b.bkey, cbegin, b.block_from,
                                                                    b.block_labels, clen, ckey, cid);
  ChunkSlices s;
  if (const int rc = slice_chunks(g, b, nb, per_block, nc, ckey, cid, clen, false, s)) return rc;
  g.block_slice_first.assign(1, 0);
  g.block_lo.clear();
  b.launched_of.assign(nb, ~0u);
  for (uint64_t q = 0; q < nb; ++q)
    if (s.slice_first[q + 1] > s.slice_first[q]) {
      b.launched_of[q] = static_cast<uint32_t>(g.block_lo.size());
      g.block_slice_first.push_back(s.slice_first[q + 1]);
      g.block_lo.push_back(static_cast<uint32_t>(b.block_from + q * b.block_labels));
    }
  const uint64_t ns = g.block_slices = s.slices;
  g.bslice_colbase = s.colbase;
  MGB_CUDA(keep_alloc(g, &g.block_idx, s.total_cols * kSliceRows));
  MGB_CUDA(keep_alloc(g, &g.block_slot, ns * kSliceRows));
  block_fill_kernel<<<blocks_for(ns * 32, g.sm_count, 16), kThreads, 0, st>>>(
      ns, s.slice_group, s.d_slice_first, s.chunk_first, g.bslice_colbase, s.sorted_id, cbegin, clen, crow, b.bkey,
      b.block_ptr, b.chunk_of, g.seg_first, static_cast<uint32_t>(g.n), g.block_idx, g.block_slot);
  return MGB200_OK;
}

// 10. SELL staging: the SELL entries whose source lies in a block with a pass become slots of stage_val, which that
// pass fills while the block is in L2, so the walk reads them in slot order instead of one random HBM sector each.
// The slots are ordered by (block, position in sell_idx); sell_idx is column-major per slice, so a column's lanes
// read neighbouring slots.  Bit 31 marks a slot: plain labels only (no hot flags), n < 2^31, fewer than 2^31 slots;
// the stream kernel reads raw labels.  The add order inside a row does not change.  By default only where the vector
// is larger than L2: where it fits, the walk's gathers from the blocks hit L2 anyway and the copy is pure cost (RMAT-22
// Katz, 32 MB on an H100's 50 MB L2: 1.4 % slower per iteration with staging, DESIGN.md §4).
int sell_staging(Graph &g, Build &b) {
  const cudaStream_t st = g.stream;
  const uint64_t n = g.n;
  const bool stage_wanted = g.tun.sell_stage > 0 || (g.tun.sell_stage < 0 && (n + 1) * sizeof(double) > b.l2_bytes);
  const bool stage_on = stage_wanted && !b.launched_of.empty() && g.sell_entries > 0 && !g.idx_flagged &&
                        !g.tun.stream_kernel && n < (1ull << 31) && g.sell_entries < (1ull << kStagePosBits);
  if (!stage_on) return MGB200_OK;
  const uint64_t ent = g.sell_entries;
  const uint32_t nl = static_cast<uint32_t>(g.block_lo.size());
  uint32_t *d_launched = nullptr;
  MGB_CUDA(b.tmp.alloc(&d_launched, b.launched_of.size()));
  MGB_CUDA(cudaMemcpyAsync(d_launched, b.launched_of.data(), b.launched_of.size() * sizeof(uint32_t),
                           cudaMemcpyHostToDevice, st));
  const StageKey stage_key{g.sell_idx, d_launched, b.block_from, b.block_labels, n};
  cub::TransformInputIterator<uint64_t, StageKey, cub::CountingInputIterator<uint64_t>> keys_in(
      cub::CountingInputIterator<uint64_t>(0), stage_key);
  cub::TransformInputIterator<uint64_t, IsStaged, decltype(keys_in)> staged_in(keys_in, IsStaged{});
  unsigned long long *d_count = nullptr;
  MGB_CUDA(b.tmp.alloc(&d_count, 1));
  MGB_CUDA(cub_call(b.tmp, [&](void *t, size_t &bytes) {
    return cub::DeviceReduce::Sum(t, bytes, staged_in, d_count, static_cast<int64_t>(ent), st);
  }));
  unsigned long long count = 0;
  MGB_CUDA(cudaMemcpyAsync(&count, d_count, sizeof(count), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  if (count == 0 || count >= (1ull << 31)) return MGB200_OK;  // the entries keep their labels
  uint64_t *skey = nullptr, *skey_alt = nullptr;
  MGB_CUDA(b.tmp.alloc(&skey, count));
  MGB_CUDA(b.tmp.alloc(&skey_alt, count));
  MGB_CUDA(cub_call(b.tmp, [&](void *t, size_t &bytes) {
    return cub::DeviceSelect::If(t, bytes, keys_in, skey, d_count, static_cast<int64_t>(ent), IsStaged{}, st);
  }));
  // positions ascend already: a stable sort on the block bits alone gives (block, position) order
  cub::DoubleBuffer<uint64_t> kb(skey, skey_alt);
  const int end_bit = kStagePosBits + bits_for(nl);
  MGB_CUDA(cub_call(b.tmp, [&](void *t, size_t &bytes) {
    return cub::DeviceRadixSort::SortKeys(t, bytes, kb, count, kStagePosBits, end_bit, st);
  }));
  MGB_CUDA(keep_alloc(g, &g.stage_src, count));
  MGB_CUDA(keep_alloc(g, &g.stage_val, count));
  stage_fill_kernel<<<blocks_for(count, g.sm_count, 16), kThreads, 0, st>>>(count, kb.Current(), g.sell_idx, g.stage_src);
  uint64_t *d_first = nullptr;
  MGB_CUDA(b.tmp.alloc(&d_first, nl + 1));
  stage_first_kernel<<<(nl + 1 + kThreads - 1) / kThreads, kThreads, 0, st>>>(nl, count, kb.Current(), d_first);
  g.stage_first.resize(nl + 1);
  MGB_CUDA(cudaMemcpyAsync(g.stage_first.data(), d_first, (nl + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  g.stage_entries = count;
  return MGB200_OK;
}

}  // namespace

int narrow_edges_u64_to_u32(int device, cudaStream_t stream, uint64_t n, uint64_t count, const uint64_t *d_in,
                            uint32_t *d_out, int *d_bad_flag) {
  MGB_CUDA(cudaSetDevice(device));
  if (count == 0) return MGB200_OK;
  int sm_count = 0;
  MGB_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device));
  narrow_kernel<<<blocks_for(count, sm_count, 16), kThreads, 0, stream>>>(count, n, d_in, d_out, d_bad_flag);
  MGB_CUDA(cudaGetLastError());
  return MGB200_OK;
}

void free_graph(Graph &g) {
  cudaSetDevice(g.device);
  for (int q = 0; q < kMaxPeers; ++q)
    if (g.peer_mapped[q]) cudaIpcCloseMemHandle(g.peer_mapped[q]);
  for (void *p : g.device_arrays) cudaFree(p);
  if (g.out_stage) cudaFree(g.out_stage);
  if (g.host_state) cudaFreeHost(g.host_state);
  for (auto &e : g.ev)
    if (e) cudaEventDestroy(e);
  for (auto &e : g.kev)
    if (e) cudaEventDestroy(e);
  if (g.fork_ev) cudaEventDestroy(g.fork_ev);
  if (g.join_ev) cudaEventDestroy(g.join_ev);
  if (g.stream2) cudaStreamDestroy(g.stream2);
  if (g.cold_fork_ev) cudaEventDestroy(g.cold_fork_ev);
  if (g.cold_join_ev) cudaEventDestroy(g.cold_join_ev);
  if (g.cold_stream) cudaStreamDestroy(g.cold_stream);
  if (g.stream) cudaStreamDestroy(g.stream);
}

int build_graph(Graph &g, EdgeSource &edges) {
  MGB_CUDA(cudaSetDevice(g.device));
  cudaDeviceProp prop{};
  MGB_CUDA(cudaGetDeviceProperties(&prop, g.device));
  g.sm_count = prop.multiProcessorCount;
  if (const int rc = open_streams(g)) return rc;
  read_tunables(g, edges.weighted());
  if (const int rc = setup_sell_table_kernel(g.device, &g.tun.table_max_bytes)) return rc;
  for (auto &e : g.ev) MGB_CUDA(cudaEventCreate(&e));
  MGB_CUDA(cudaEventRecord(g.ev[0], g.stream));
  Build b{edges, edges.weighted(), static_cast<uint64_t>(prop.l2CacheSize), Dealer{g.n, g.part_world}};
  map_rows(g, b);
  if (const int rc = iteration_state(g)) return rc;
  if (g.n == 0) {
    MGB_CUDA(keep_alloc(g, &g.rank, 0));
    MGB_CUDA(keep_alloc(g, &g.local_vertex, 0));
    MGB_CUDA(cudaEventRecord(g.ev[1], g.stream));
    MGB_CUDA(cudaStreamSynchronize(g.stream));
    return MGB200_OK;
  }
  if (const int rc = labels(g, b)) return rc;
  if (const int rc = row_classes(g, b)) return rc;
  if (const int rc = edge_keys(g, b)) return rc;
  if (const int rc = row_pointers(g, b)) return rc;
  if (const int rc = block_edges(g, b)) return rc;
  if (g.n_heavy) {
    if (const int rc = heavy_class(g, b)) return rc;
    if (const int rc = tile_slices(g, b)) return rc;
    note_mem(g);
  }
  if (const int rc = sell_class(g, b)) return rc;
  if (const int rc = block_slices(g, b)) return rc;
  if (const int rc = sell_staging(g, b)) return rc;
  note_mem(g);
  MGB_CUDA(cudaGetLastError());
  MGB_CUDA(cudaEventRecord(g.ev[1], g.stream));
  MGB_CUDA(cudaStreamSynchronize(g.stream));
  float ms = 0.f;
  MGB_CUDA(cudaEventElapsedTime(&ms, g.ev[0], g.ev[1]));
  g.build_ms = ms;
  return MGB200_OK;
}

}  // namespace mgb200

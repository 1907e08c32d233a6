// memgraph_b200/csrc/hits.cu -- HITS hubs and authorities (cuGraph semantics) on two PageRank graph layouts of one COO;
// include/mgb200_personalized.h has the recurrence and the reference call site.
//
// The forward handle F (edges u -> v) gathers along in-edges: auth = A^T hubs.  The reverse handle T (the same COO with
// the endpoints swapped) gathers along F's out-edges: hubs = A auth.  Both gathers are PageRank's (launch_gather_phase:
// SELL row sums, heavy row sums, same cache policies); the two handles sort their labels by different degrees, so the
// vectors cross between the label spaces through two permutations built once per graph:
//   t_of_f[l] = T label of the vertex with F label l,   f_of_t[l] = F label of the vertex with T label l.
// One iteration (every kernel on F's stream until the gather of T, whose stream waits on an event, and back):
//   F gather over contrib_F (hubs by F label)            -> auth by F row
//   max over F rows; contrib_T[t_of_f[r]] = auth[r] / max  (authority epilogue)
//   T gather over contrib_T                              -> hubs by T row
//   max over T rows; h = hubs[r] / max; diff += |h - prev[r]|; prev[r] = h; contrib_F[f_of_t[r]] = h   (hub epilogue)
//   one 8-byte copy of diff for the host's stop test
// Every reduction is two-stage with a fixed tree (per-block partials of a fixed chunk, then one block), so results are
// bit-reproducible run to run; a maximum is exact in any order.  One partition: label == local row on each handle.
#include <algorithm>

#include "core.hpp"
#include "mgb200_personalized.h"

namespace mgb200 {
namespace {

constexpr int kPartials = 1024;

// one block per 4 * kThreads items, at most kPartials: the partials buffer holds one value per block
inline int partial_blocks(uint64_t items) {
  return static_cast<int>(std::max<uint64_t>(1, std::min<uint64_t>((items + kThreads * 4 - 1) / (kThreads * 4), kPartials)));
}

struct OpSum {
  __device__ static double apply(double a, double b) { return a + b; }
};
struct OpMax {
  __device__ static double apply(double a, double b) { return fmax(a, b); }
};

template <typename Op>
__device__ __forceinline__ double block_reduce(double v) {
  __shared__ double sm[kThreads];
  sm[threadIdx.x] = v;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sm[threadIdx.x] = Op::apply(sm[threadIdx.x], sm[threadIdx.x + o]);
    __syncthreads();
  }
  return sm[0];
}

// The gathered sums of one handle by row: heavy rows, SELL rows, then rows without in-edges (0).
struct RowSums {
  uint64_t n, n_heavy, n_sell;
  const double *heavy, *sell;
  __device__ __forceinline__ double at(uint64_t r) const {
    return r < n_heavy ? heavy[r] : (r < n_heavy + n_sell ? sell[r - n_heavy] : 0.0);
  }
};

RowSums row_sums(const Graph &g) { return RowSums{g.n, g.n_heavy, g.n_sell, g.heavy_sums, g.sell_sums}; }

__global__ void __launch_bounds__(kThreads) hits_init_kernel(uint64_t n, double *contrib_f, double *contrib_t,
                                                             double *hubs_t, IterState *state_f, IterState *state_t) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const double h0 = 1.0 / static_cast<double>(n);
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    contrib_f[i] = h0;  // uniform: the same in every label order
    hubs_t[i] = h0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    contrib_f[n] = 0.0;  // the slot SELL padding entries read
    contrib_t[n] = 0.0;
    state_f->done = 0;   // the gather kernels return at once while this is set
    state_f->error = 0;
    state_t->done = 0;
    state_t->error = 0;
  }
}

// block b owns one contiguous chunk of rows, so the partials do not depend on the grid's timing
__global__ void __launch_bounds__(kThreads) row_max_kernel(RowSums s, double *partials) {
  const uint64_t chunk = (s.n + gridDim.x - 1) / gridDim.x;
  const uint64_t lo = chunk * blockIdx.x, hi = min(lo + chunk, s.n);
  double mx = 0.0;
  for (uint64_t r = lo + threadIdx.x; r < hi; r += blockDim.x) mx = fmax(mx, s.at(r));
  const double b = block_reduce<OpMax>(mx);
  if (threadIdx.x == 0) partials[blockIdx.x] = b;
}

__global__ void __launch_bounds__(kThreads) vec_sum_kernel(uint64_t n, const double *v, double *partials) {
  const uint64_t chunk = (n + gridDim.x - 1) / gridDim.x;
  const uint64_t lo = chunk * blockIdx.x, hi = min(lo + chunk, n);
  double acc = 0.0;
  for (uint64_t r = lo + threadIdx.x; r < hi; r += blockDim.x) acc += v[r];
  const double b = block_reduce<OpSum>(acc);
  if (threadIdx.x == 0) partials[blockIdx.x] = b;
}

template <typename Op>
__global__ void __launch_bounds__(kThreads) reduce_kernel(const double *partials, int count, double *out) {
  double acc = 0.0;  // identity of both: the maxima and sums here are over values >= 0
  for (int i = threadIdx.x; i < count; i += blockDim.x) acc = Op::apply(acc, partials[i]);
  const double s = block_reduce<Op>(acc);
  if (threadIdx.x == 0) *out = s;
}

// authority epilogue: auth by F row, scaled by its maximum, into T's label space
__global__ void __launch_bounds__(kThreads) auth_scatter_kernel(RowSums s, const double *max_auth,
                                                                const uint32_t *t_of_f, double *contrib_t) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const double mx = *max_auth;
  for (uint64_t r = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < s.n; r += stride)
    contrib_t[t_of_f[r]] = s.at(r) / mx;
}

// hub epilogue: hubs by T row, scaled by their maximum; L1 distance to the previous hubs (T order, updated in place);
// the new hubs into F's label space for the next iteration
__global__ void __launch_bounds__(kThreads) hub_epilogue_kernel(RowSums s, const double *max_hubs,
                                                                const uint32_t *f_of_t, double *hubs_t,
                                                                double *contrib_f, double *partials) {
  const uint64_t chunk = (s.n + gridDim.x - 1) / gridDim.x;
  const uint64_t lo = chunk * blockIdx.x, hi = min(lo + chunk, s.n);
  const double mx = *max_hubs;
  double diff = 0.0;
  for (uint64_t r = lo + threadIdx.x; r < hi; r += blockDim.x) {
    const double h = s.at(r) / mx;
    diff += fabs(h - hubs_t[r]);
    hubs_t[r] = h;
    contrib_f[f_of_t[r]] = h;
  }
  const double b = block_reduce<OpSum>(diff);
  if (threadIdx.x == 0) partials[blockIdx.x] = b;
}

// both vectors are held by T label; sums = nullptr: not normalised
__global__ void __launch_bounds__(kThreads) hits_write_kernel(uint64_t n, const uint32_t *label_of_t, const double *hubs_t,
                                                              const double *auth_t, const double *sums, double *hubs_out,
                                                              double *auth_out) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const double hs = sums ? sums[0] : 1.0, as = sums ? sums[1] : 1.0;
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n; v += stride) {
    const uint32_t l = label_of_t[v];
    hubs_out[v] = sums ? hubs_t[l] / hs : hubs_t[l];
    auth_out[v] = sums ? auth_t[l] / as : auth_t[l];
  }
}

__global__ void __launch_bounds__(kThreads) permutation_kernel(uint64_t n, const uint32_t *local_vertex_a,
                                                               const uint32_t *label_of_b, uint32_t *b_of_a) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t l = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; l < n; l += stride)
    b_of_a[l] = label_of_b[local_vertex_a[l]];
}

}  // namespace

int hits_permutations(Graph &f, Graph &t, uint32_t *t_of_f, uint32_t *f_of_t) {
  MGB_CUDA(cudaSetDevice(f.device));
  if (f.n == 0) return MGB200_OK;
  // T's build finished on T's stream; F's label arrays were final before it started
  MGB_CUDA(cudaStreamSynchronize(t.stream));
  permutation_kernel<<<partial_blocks(f.n), kThreads, 0, f.stream>>>(f.n, f.local_vertex, t.label_of, t_of_f);
  permutation_kernel<<<partial_blocks(f.n), kThreads, 0, f.stream>>>(f.n, t.local_vertex, f.label_of, f_of_t);
  MGB_CUDA(cudaGetLastError());
  MGB_CUDA(cudaStreamSynchronize(f.stream));
  return MGB200_OK;
}

// d_hubs / d_auth: n doubles each on the device, original vertex order.  `scratch`: hits_scratch_doubles(n) doubles.
uint64_t hits_scratch_doubles(uint64_t n) { return n + kPartials + 4; }

int hits_iterate(Graph &f, Graph &t, const uint32_t *t_of_f, const uint32_t *f_of_t, const mgb200_hits_params &prm,
                 double *scratch, cudaEvent_t f_done, cudaEvent_t t_done, double *d_hubs, double *d_auth,
                 mgb200_hits_stats *stats) {
  MGB_CUDA(cudaSetDevice(f.device));
  const uint64_t n = f.n;
  *stats = mgb200_hits_stats{};
  stats->converged = 1;
  if (n == 0) return MGB200_OK;
  cudaStream_t fs = f.stream, ts = t.stream;
  double *hubs_t = scratch;                // [n] previous / current hubs by T row
  double *partials = scratch + n;          // [kPartials]
  double *scalars = partials + kPartials;  // [0] max auth, [1] max hubs, [2] diff, [3] spare
  double *contrib_f = f.contrib(0), *contrib_t = t.contrib(0);
  const int blocks = partial_blocks(n);
  uint64_t launches = 0;
  if (f.m == 0) {  // no edge: every score is 0 (the divisions by the maxima below need an edge)
    MGB_CUDA(cudaMemsetAsync(d_hubs, 0, n * sizeof(double), fs));
    MGB_CUDA(cudaMemsetAsync(d_auth, 0, n * sizeof(double), fs));
    MGB_CUDA(cudaStreamSynchronize(fs));
    return MGB200_OK;
  }
  MGB_CUDA(cudaEventRecord(f.ev[2], fs));
  hits_init_kernel<<<blocks, kThreads, 0, fs>>>(n, contrib_f, contrib_t, hubs_t, f.state, t.state);
  ++launches;
  const RowSums sf = row_sums(f), st = row_sums(t);
  uint64_t it = 0;
  int converged = 0;
  double diff_host = 0.0;
  const double stop = static_cast<double>(n) * prm.tolerance;
  while (true) {
    // authorities: F's gather over the hubs, then the epilogue into T's labels
    int rc = launch_gather_phase(f, contrib_f, &launches, /*heavy_row_sums=*/true);
    if (rc) return rc;
    row_max_kernel<<<blocks, kThreads, 0, fs>>>(sf, partials);
    reduce_kernel<OpMax><<<1, kThreads, 0, fs>>>(partials, blocks, scalars);
    auth_scatter_kernel<<<blocks, kThreads, 0, fs>>>(sf, scalars, t_of_f, contrib_t);
    launches += 3;
    MGB_CUDA(cudaEventRecord(f_done, fs));
    MGB_CUDA(cudaStreamWaitEvent(ts, f_done, 0));
    // hubs: T's gather over the authorities, then the epilogue into F's labels
    rc = launch_gather_phase(t, contrib_t, &launches, /*heavy_row_sums=*/true);
    if (rc) return rc;
    row_max_kernel<<<blocks, kThreads, 0, ts>>>(st, partials);
    reduce_kernel<OpMax><<<1, kThreads, 0, ts>>>(partials, blocks, scalars + 1);
    hub_epilogue_kernel<<<blocks, kThreads, 0, ts>>>(st, scalars + 1, f_of_t, hubs_t, contrib_f, partials);
    reduce_kernel<OpSum><<<1, kThreads, 0, ts>>>(partials, blocks, scalars + 2);
    launches += 4;
    MGB_CUDA(cudaMemcpyAsync(&diff_host, scalars + 2, sizeof(double), cudaMemcpyDeviceToHost, ts));
    MGB_CUDA(cudaEventRecord(t_done, ts));
    MGB_CUDA(cudaStreamWaitEvent(fs, t_done, 0));
    MGB_CUDA(cudaStreamSynchronize(ts));
    ++it;
    if (diff_host < stop) {
      converged = 1;
      break;
    }
    if (it >= prm.max_iterations) break;
  }
  // the last hubs (hubs_t) and authorities (contrib_t) are both held by T label; F's stream waits on T's already
  const double *sums = nullptr;
  if (prm.normalized) {
    vec_sum_kernel<<<blocks, kThreads, 0, fs>>>(n, hubs_t, partials);
    reduce_kernel<OpSum><<<1, kThreads, 0, fs>>>(partials, blocks, scalars);
    vec_sum_kernel<<<blocks, kThreads, 0, fs>>>(n, contrib_t, partials);
    reduce_kernel<OpSum><<<1, kThreads, 0, fs>>>(partials, blocks, scalars + 1);
    launches += 4;
    sums = scalars;
  }
  hits_write_kernel<<<partial_blocks(n), kThreads, 0, fs>>>(n, t.label_of, hubs_t, contrib_t, sums, d_hubs, d_auth);
  ++launches;
  MGB_CUDA(cudaEventRecord(f.ev[3], fs));
  MGB_CUDA(cudaStreamSynchronize(fs));
  MGB_CUDA(cudaGetLastError());
  float ms = 0.f;
  MGB_CUDA(cudaEventElapsedTime(&ms, f.ev[2], f.ev[3]));
  stats->iterations = it;
  stats->converged = converged;
  stats->last_diff_sum = diff_host;
  stats->iterate_ms = ms;
  stats->kernel_launches = launches;
  return MGB200_OK;
}

}  // namespace mgb200

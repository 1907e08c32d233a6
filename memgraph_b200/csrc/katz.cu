// memgraph_b200/csrc/katz.cu -- static Katz centrality on the PageRank graph layout (SURVEY 8f-1).
//
// Restates katz_alg::SetKatz / KatzCentralityLoop / Converged
// (mage/cpp/katz_centrality_module/algorithm/katz.cpp:389-410, :222-251, :163-211) as device work:
//   * omega_i = A^T omega_{i-1} is PageRank's gather phase verbatim (launch_gather_phase: SELL row sums + heavy segment
//     partials, same cache policies) over the omega vector instead of the contribution vector; the two omega buffers
//     ARE the graph handle's two contribution buffers, c lives in its rank array;
//   * the row epilogue applies c += alpha^i omega, ur = c + alpha^(i+1) omega gamma with the reference's association
//     and one rounding per operation (no FMA contraction: the reference is compiled for baseline x86-64);
//   * zero in-degree rows: omega_i = 0 for i >= 1, so c = 0 and ur = 0 + 0 * gamma forever -- set once, never
//     visited.  That ur is +0 while gamma is finite and NaN when alpha^2 deg_max == 1 makes gamma = +inf; NaN fails
//     every comparison, so with epsilon <= 0 these rows still let the test pass, exactly as in the reference;
//   * the convergence test sorts (c descending) with a radix sort and decides from neighbour pairs.  The reference
//     sorts with std::partial_sort, which is unstable; the verdict is independent of the order among equal c except
//     when a group of equal-c vertices contains EXACTLY ONE vertex whose own bound already violates the test against an
//     equal predecessor (see verdict kernels).  Only then is partial_sort's actual permutation replayed
//     (katz_heap.hpp, one device thread) -- never the CPU.
// alpha^i comes from the host's pow(), the same libm call the reference makes (:236, :244).
#include <cmath>
#include <cub/cub.cuh>

#include "core.hpp"
#include "katz_heap.hpp"
#include "mgb200_katz.h"

namespace mgb200 {
namespace {

struct Verdict {
  unsigned int definite_fail;  // some neighbour pair violates the test under EVERY order of equal centralities
  unsigned int ambiguous;      // groups of equal c with exactly one self-violating member and at least two members
  unsigned int tie_mismatch;   // ambiguous groups whose self-violating member is NOT first in partial_sort's order
  unsigned int max_outdeg;
};

// context.Init (:33-45): omega_0 = 1, c_0 = 0; omega_1 of the zero in-degree rows is their final value 0.  Those rows
// are never visited again, so their ur is written here once: the reference's c + (alpha^(i+1) * 0) * gamma, which is
// zero_ur = 0 + 0 * gamma at every iteration -- +0 while gamma is finite, NaN when it is not (alpha^2 deg_max == 1).
__global__ void katz_init_kernel(uint64_t n, uint64_t zero_lo, uint64_t zero_hi, double zero_ur, double *omega0,
                                 double *omega1, double *c, double *ur, IterState *state) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    omega0[i] = 1.0;
    omega1[i] = 0.0;
    c[i] = 0.0;
    ur[i] = (i >= zero_lo && i < zero_hi) ? zero_ur : 0.0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    omega0[n] = 0.0;  // the slot SELL padding entries read
    omega1[n] = 0.0;
    state->done = 0;  // the gather kernels return at once while this is set
    state->error = 0;
    state->iterations = 0ull;
  }
}

__global__ void fill_zero_kernel(uint64_t lo, uint64_t hi, double *v) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = lo + static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < hi; i += stride) v[i] = 0.0;
}

// MaxDegree (:133-143)
__global__ void max_outdeg_kernel(uint64_t n, const uint32_t *outdeg, Verdict *verdict) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  unsigned int m = 0;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    m = max(m, outdeg[i]);
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(&verdict->max_outdeg, m);
}

struct KatzStep {
  double a_i;     // alpha^iteration
  double a_next;  // alpha^(iteration + 1)
  double gamma;
  double *omega_out;  // [n + 1] by label (one partition: label == local row)
  double *c;          // [n] in place
  double *ur;         // [n]
};

// :233-245 for one row whose gathered sum is w
__device__ __forceinline__ void katz_row(const KatzStep &k, uint64_t row, double w) {
  k.omega_out[row] = w;
  const double cn = __dadd_rn(k.c[row], __dmul_rn(k.a_i, w));
  k.c[row] = cn;
  k.ur[row] = __dadd_rn(cn, __dmul_rn(__dmul_rn(k.a_next, w), k.gamma));  // (pow * omega) * gamma, then the sum
}

__global__ void katz_sell_epilogue_kernel(uint64_t first_row, uint64_t end_row, const double *sums, KatzStep k) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t r = first_row + static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < end_row; r += stride)
    katz_row(k, r, sums[r - first_row]);
}

// warp per heavy row: segment partials summed in segment order with the same shuffle tree as PageRank's finish
__global__ void katz_heavy_finish_kernel(uint64_t n_heavy, const uint64_t *seg_first, const double *seg_partial,
                                         KatzStep k) {
  const int lane = threadIdx.x & 31;
  const uint64_t warps_total = static_cast<uint64_t>(gridDim.x) * (blockDim.x >> 5);
  for (uint64_t r = static_cast<uint64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n_heavy;
       r += warps_total) {
    const uint64_t s0 = seg_first[r], s1 = seg_first[r + 1];
    double acc = 0.0;
    for (uint64_t s = s0 + lane; s < s1; s += 32) acc += seg_partial[s];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if (lane == 0) katz_row(k, r, acc);
  }
}

// ---- Converged (:163-211), k = number of vertices (:170) ---------------------------------------------------------
//
// Sorted by c descending, positions [s, e) with equal c form a group.  A member b at position i is tested against its
// predecessor a:  NOT converged if  ur[b] - eps >= lr[a] = c[a].
//   * predecessor in the SAME group (c[a] == c[b]):      "strict" test   ur[b] - eps >= c[b]
//   * b first of its group (predecessor = previous group): "weak" test   ur[b] - eps >= c[previous group]  (> c[b])
// A member that fails the weak test fails the strict one too.  Hence, whatever the order inside groups:
//   some member fails weak                      -> not converged
//   some group has >= 2 strict-failing members  -> not converged (at most one of them can be first)
//   no member fails strict                      -> converged
// and otherwise (groups with exactly ONE strict-failing member, which passes weak) the verdict is "converged iff that
// member is the first of its group in partial_sort's order" -- the only case that needs the real permutation.

__global__ void iota_keys_kernel(uint64_t n, const double *c, double *key, uint32_t *val) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    key[i] = c[i];
    val[i] = static_cast<uint32_t>(i);
  }
}

__global__ void group_mark_kernel(uint64_t n, const double *key_sorted, uint32_t *start_or_zero, uint32_t *strict_count,
                                  Verdict *verdict) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    start_or_zero[i] = (i > 0 && key_sorted[i - 1] != key_sorted[i]) ? static_cast<uint32_t>(i) : 0u;
    strict_count[i] = 0u;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    verdict->definite_fail = 0u;
    verdict->ambiguous = 0u;
    verdict->tie_mismatch = 0u;
  }
}

// group_start[i] = first position of i's group (inclusive max-scan of start_or_zero)
__global__ void member_test_kernel(uint64_t n, const double *key_sorted, const uint32_t *row_sorted,
                                   const uint32_t *group_start, const double *ur, double eps, uint32_t *strict_count,
                                   uint32_t *strict_row, Verdict *verdict) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t row = row_sorted[i];
    const uint32_t s = group_start[i];
    const double bound = __dsub_rn(ur[row], eps);
    if (s > 0 && bound >= key_sorted[s - 1]) verdict->definite_fail = 1u;  // fails even as the first of its group
    if (bound >= key_sorted[i]) {
      atomicAdd(strict_count + s, 1u);
      strict_row[s] = row;  // meaningful only when the count ends at 1
    }
  }
}

__global__ void group_verdict_kernel(uint64_t n, const uint32_t *group_start, const uint32_t *strict_count,
                                     Verdict *verdict) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (group_start[i] != i) continue;  // group starts only
    const uint32_t cnt = strict_count[i];
    const bool several_members = i + 1 < n && group_start[i + 1] == i;
    if (cnt >= 2) verdict->definite_fail = 1u;
    if (cnt == 1 && several_members) atomicAdd(&verdict->ambiguous, 1u);
  }
}

// ---- the rare path: replay std::partial_sort's permutation (ids ascending on entry, :174-177) ---------------------

__global__ void c_by_vertex_kernel(uint64_t n, const uint32_t *label_of, const double *c, double *c_by_vertex,
                                   uint32_t *order) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n; v += stride) {
    c_by_vertex[v] = c[label_of[v]];
    order[v] = static_cast<uint32_t>(v);
  }
}

__global__ void tie_order_kernel(uint64_t n, uint32_t *order, const double *c_by_vertex) {
  if (blockIdx.x == 0 && threadIdx.x == 0) KatzTieOrder::run(order, static_cast<int64_t>(n), c_by_vertex);
}

// partial_sort's order and the radix order agree on which positions every group occupies (both are sorted by c)
__global__ void tie_check_kernel(uint64_t n, const uint32_t *group_start, const uint32_t *strict_count,
                                 const uint32_t *strict_row, const uint32_t *order, const uint32_t *label_of,
                                 Verdict *verdict) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (group_start[i] != i || strict_count[i] != 1u) continue;
    if (!(i + 1 < n && group_start[i + 1] == i)) continue;
    if (label_of[order[i]] != strict_row[i]) atomicAdd(&verdict->tie_mismatch, 1u);
  }
}

__global__ void write_by_vertex_kernel(uint64_t n, const uint32_t *label_of, const double *c, double *out) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < n; v += stride)
    out[v] = c[label_of[v]];
}

struct MaxOp {
  __host__ __device__ uint32_t operator()(uint32_t a, uint32_t b) const { return a > b ? a : b; }
};

}  // namespace

int katz_iterate(Graph &g, double alpha, double epsilon, uint64_t max_iterations, double *d_out, KatzResult *res) {
  *res = KatzResult{};
  if (g.part_world != 1) {
    set_error("Katz centrality runs on a single partition (part_world == 1)");
    return MGB200_ERR_INVALID_ARGUMENT;
  }
  MGB_CUDA(cudaSetDevice(g.device));
  cudaStream_t st = g.stream;
  const uint64_t n = g.n;
  if (n == 0) {
    res->converged = true;
    return MGB200_OK;
  }
  if (g.m == 0) {  // :395-397: no edges, every centrality is c_0 = 0
    MGB_CUDA(cudaMemsetAsync(d_out, 0, n * sizeof(double), st));
    MGB_CUDA(cudaStreamSynchronize(st));
    res->converged = true;
    return MGB200_OK;
  }
  DeviceBuffers tmp;
  double *ur = nullptr, *key = nullptr, *key_alt = nullptr, *c_by_vertex = nullptr;
  uint32_t *val = nullptr, *val_alt = nullptr, *start = nullptr, *strict_count = nullptr, *strict_row = nullptr,
           *order = nullptr;
  Verdict *verdict = nullptr;
  MGB_CUDA(tmp.alloc(&ur, n));
  MGB_CUDA(tmp.alloc(&key, n));
  MGB_CUDA(tmp.alloc(&key_alt, n));
  MGB_CUDA(tmp.alloc(&val, n));
  MGB_CUDA(tmp.alloc(&val_alt, n));
  MGB_CUDA(tmp.alloc(&start, n));
  MGB_CUDA(tmp.alloc(&strict_count, n));
  MGB_CUDA(tmp.alloc(&strict_row, n));
  MGB_CUDA(tmp.alloc(&verdict, 1));
  size_t sort_bytes = 0, scan_bytes = 0;
  {
    cub::DoubleBuffer<double> kb(key, key_alt);
    cub::DoubleBuffer<uint32_t> vb(val, val_alt);
    MGB_CUDA(cub::DeviceRadixSort::SortPairsDescending(nullptr, sort_bytes, kb, vb, n, 0, 64, st));
    MGB_CUDA(cub::DeviceScan::InclusiveScan(nullptr, scan_bytes, start, start, MaxOp(), n, st));
  }
  char *cub_tmp = nullptr;
  MGB_CUDA(tmp.alloc(&cub_tmp, std::max(sort_bytes, scan_bytes)));
  const size_t cub_bytes = std::max(sort_bytes, scan_bytes);

  double *omega[2] = {g.contrib(0), g.contrib(1)};
  double *c = g.rank;  // one partition: local_rows == n and label == local row
  const int grid_n = blocks_for(n, g.sm_count, 16);

  MGB_CUDA(cudaEventRecord(g.ev[2], st));
  MGB_CUDA(cudaMemsetAsync(verdict, 0, sizeof(Verdict), st));
  max_outdeg_kernel<<<grid_n, kThreads, 0, st>>>(n, g.outdeg_l, verdict);
  Verdict host_verdict{};
  MGB_CUDA(cudaMemcpyAsync(&host_verdict, verdict, sizeof(Verdict), cudaMemcpyDeviceToHost, st));
  MGB_CUDA(cudaStreamSynchronize(st));
  const double deg_max = static_cast<double>(host_verdict.max_outdeg);
  const double gamma = deg_max / (1. - (alpha * alpha * deg_max));  // :400
  res->max_out_degree = host_verdict.max_outdeg;
  res->gamma = gamma;

  const uint64_t zero_lo = g.zero_lo[0], zero_hi = g.zero_hi[0];  // labels of the zero in-degree rows
  const double zero_ur = 0.0 + 0.0 * gamma;  // :245 with omega = 0, whatever the sign of alpha^(i+1)
  katz_init_kernel<<<grid_n, kThreads, 0, st>>>(n, zero_lo, zero_hi, zero_ur, omega[0], omega[1], c, ur, g.state);
  uint64_t launches = 2;
  uint64_t iteration = 0;
  bool converged = false;
  do {
    ++iteration;
    KatzStep k{};
    k.a_i = pow(alpha, static_cast<double>(iteration));
    k.a_next = pow(alpha, static_cast<double>(iteration + 1));
    k.gamma = gamma;
    k.omega_out = omega[iteration & 1ull];
    k.c = c;
    k.ur = ur;
    const double *omega_in = omega[(iteration - 1) & 1ull];
    int rc = launch_gather_phase(g, omega_in, &launches);
    if (rc) return rc;
    if (g.n_sell) {
      const uint64_t r0 = g.n_heavy, r1 = g.n_heavy + g.n_sell;
      katz_sell_epilogue_kernel<<<blocks_for(r1 - r0, g.sm_count, 16), kThreads, 0, st>>>(r0, r1, g.sell_sums, k);
      ++launches;
    }
    if (g.n_heavy) {
      katz_heavy_finish_kernel<<<blocks_for(g.n_heavy * 32, g.sm_count, 16), kThreads, 0, st>>>(g.n_heavy, g.seg_first,
                                                                                            g.seg_partial, k);
      ++launches;
    }
    if (iteration == 2 && zero_hi > zero_lo) {  // buffer 0 still holds omega_0 = 1 for the rows nobody visits
      fill_zero_kernel<<<blocks_for(zero_hi - zero_lo, g.sm_count, 16), kThreads, 0, st>>>(zero_lo, zero_hi, omega[0]);
      ++launches;
    }
    // Converged(): sort by c descending, then the neighbour tests
    iota_keys_kernel<<<grid_n, kThreads, 0, st>>>(n, c, key, val);
    cub::DoubleBuffer<double> kb(key, key_alt);
    cub::DoubleBuffer<uint32_t> vb(val, val_alt);
    size_t bytes = cub_bytes;
    MGB_CUDA(cub::DeviceRadixSort::SortPairsDescending(cub_tmp, bytes, kb, vb, n, 0, 64, st));
    const double *key_sorted = kb.Current();
    const uint32_t *row_sorted = vb.Current();
    group_mark_kernel<<<grid_n, kThreads, 0, st>>>(n, key_sorted, start, strict_count, verdict);
    bytes = cub_bytes;
    MGB_CUDA(cub::DeviceScan::InclusiveScan(cub_tmp, bytes, start, start, MaxOp(), n, st));
    member_test_kernel<<<grid_n, kThreads, 0, st>>>(n, key_sorted, row_sorted, start, ur, epsilon, strict_count,
                                                     strict_row, verdict);
    group_verdict_kernel<<<grid_n, kThreads, 0, st>>>(n, start, strict_count, verdict);
    launches += 6;  // keys, sort, mark, scan, member test, group verdict (library launches counted once each)
    MGB_CUDA(cudaMemcpyAsync(&host_verdict, verdict, sizeof(Verdict), cudaMemcpyDeviceToHost, st));
    MGB_CUDA(cudaStreamSynchronize(st));
    converged = host_verdict.definite_fail == 0;
    if (converged && host_verdict.ambiguous != 0) {
      if (!order) {
        MGB_CUDA(tmp.alloc(&order, n));
        MGB_CUDA(tmp.alloc(&c_by_vertex, n));
      }
      c_by_vertex_kernel<<<grid_n, kThreads, 0, st>>>(n, g.label_of, c, c_by_vertex, order);
      tie_order_kernel<<<1, 32, 0, st>>>(n, order, c_by_vertex);
      tie_check_kernel<<<grid_n, kThreads, 0, st>>>(n, start, strict_count, strict_row, order, g.label_of, verdict);
      launches += 3;
      MGB_CUDA(cudaMemcpyAsync(&host_verdict, verdict, sizeof(Verdict), cudaMemcpyDeviceToHost, st));
      MGB_CUDA(cudaStreamSynchronize(st));
      converged = host_verdict.tie_mismatch == 0;
      ++res->tie_order_runs;
    }
    if (max_iterations && iteration >= max_iterations) break;  // caller's guard; the reference has none
  } while (!converged);
  write_by_vertex_kernel<<<grid_n, kThreads, 0, st>>>(n, g.label_of, c, d_out);
  ++launches;
  MGB_CUDA(cudaEventRecord(g.ev[3], st));
  MGB_CUDA(cudaStreamSynchronize(st));
  MGB_CUDA(cudaGetLastError());
  float ms = 0.f;
  MGB_CUDA(cudaEventElapsedTime(&ms, g.ev[2], g.ev[3]));
  res->iterations = iteration;
  res->launches = launches;
  res->iterate_ms = ms;
  res->converged = converged;
  return MGB200_OK;
}

}  // namespace mgb200

using namespace mgb200;

extern "C" {

int mgb200_katz_tie_order(uint64_t n, const double *keys, uint32_t *order_out) {
  if (n > 0 && (!keys || !order_out)) return MGB200_ERR_INVALID_ARGUMENT;
  if (n >= 0xFFFFFFFFull) return MGB200_ERR_INVALID_ARGUMENT;
  for (uint64_t i = 0; i < n; ++i) order_out[i] = static_cast<uint32_t>(i);
  KatzTieOrder::run(order_out, static_cast<int64_t>(n), keys);  // the same code the device runs
  return MGB200_OK;
}

}  // extern "C"

/*
 * mgb200_katz.h -- C ABI of the GPU-native STATIC Katz centrality (SURVEY 8f-1, the path after PageRank).
 *
 *   reference interface                                                    replaced by
 *   ---------------------------------------------------------------------  ---------------------------------
 *   katz_alg::SetKatz(graph, alpha = 0.2, epsilon = 1e-2)                  mgb200_katz_run() on a graph handle
 *     mage/cpp/katz_centrality_module/algorithm/katz.hpp:34-35,            built by mgb200_graph_create_*()
 *     katz.cpp:389-410 (SetKatz), :222-251 (KatzCentralityLoop),           (mgb200_pagerank.h: the same degree-
 *     :163-211 (Converged), :133-143 (MaxDegree)                           sorted SELL-32 + segmented CSC layout)
 *   both, as GetKatzCentrality calls them                                  mgb200_katz_centrality()
 *     katz_centrality_module.cpp:38-53
 *
 * What is computed (ids 0..n-1, multi-edges counted, directed):
 *   omega_0 = 1, c_0 = 0, gamma = deg_max / (1 - alpha^2 deg_max), deg_max = largest out-degree
 *   iteration i >= 1:  omega_i[v] = sum_{u -> v} omega_{i-1}[u];  c_i[v] = c_{i-1}[v] + alpha^i omega_i[v]
 *                      lr[v] = c_i[v];  ur[v] = c_i[v] + alpha^(i+1) omega_i[v] gamma
 *   stop when, walking the vertices in std::partial_sort order of c_i descending, no neighbour pair (a, b) has
 *   ur[b] - epsilon >= lr[a].  ur is computed for EVERY vertex: where omega_i[v] = 0 it is c_i[v] + 0 * gamma, NaN when
 *   alpha^2 deg_max == 1 makes gamma = +inf, and a NaN bound fails no comparison (so with epsilon <= 0 vertices without
 *   in-edges do not hold the loop).  No edges: every centrality is 0.  The reference has no iteration cap; max_iterations
 *   below is a guard for callers (0 = none) and reports MGB200_KATZ_NOT_CONVERGED when it ends the loop.
 * Parity: omega_i are walk counts -- integers, exact in FP64 below 2^53 in any summation order -- and every other
 * operation is performed with the reference's association and rounding, so results are BIT-EXACT until a walk count
 * passes 2^53 (then the summation order inside a row differs from the reference's).
 * Single partition only (part_world == 1).  No CPU fallback.
 */
#ifndef MGB200_KATZ_H
#define MGB200_KATZ_H

#include "mgb200_pagerank.h"

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

#define MGB200_KATZ_NOT_CONVERGED 16 /* max_iterations reached first; centrality_out holds the last iterate */

typedef struct mgb200_katz_stats {
  uint64_t iterations;       /* katz_alg::context.iteration at return                                   */
  uint64_t max_out_degree;   /* deg_max (:133-143)                                                      */
  double gamma;              /* :400                                                                    */
  double iterate_ms;         /* CUDA-event time of the loop (init .. last convergence test)             */
  uint64_t kernel_launches;  /* kernels launched inside the timed region                                */
  uint64_t tie_order_runs;   /* iterations whose verdict depended on partial_sort's tie order and were
                                settled by replaying that order on the device (katz_heap.hpp)          */
} mgb200_katz_stats;

/* SetKatz on a device-resident graph.  centrality_out: n doubles, HOST memory, original vertex-id order. */
int mgb200_katz_run(mgb200_graph *g, double alpha, double epsilon, uint64_t max_iterations, double *centrality_out,
                    mgb200_katz_stats *stats);

/* Graph ingest + SetKatz in one call, host buffers in and out (what GetKatzCentrality does between GetGraphView and
 * record emission, katz_centrality_module.cpp:43-44). */
int mgb200_katz_centrality(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, double alpha,
                           double epsilon, uint64_t max_iterations, double *centrality_out, uint64_t *iterations_out);

/* Host-only diagnostic: the order std::partial_sort(first, last, last, key-descending) leaves ids 0..n-1 in, computed by
 * the index-arithmetic restatement the device uses for tie-order-dependent verdicts (csrc/katz_heap.hpp). */
int mgb200_katz_tie_order(uint64_t n, const double *keys, uint32_t *order_out);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* MGB200_KATZ_H */

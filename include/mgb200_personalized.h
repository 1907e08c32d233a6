/*
 * mgb200_personalized.h -- C ABI of the cuGraph-semantics PageRank variants (SURVEY 8f-4): what the reference's
 * cugraph.pagerank.get / cugraph.personalized_pagerank.get compute, on the same device-resident layout as the in-tree
 * PageRank (mgb200_pagerank.h), so that the GPU module can stand in for the cuGraph modules too.
 *
 *   reference call site                                                        replaced by
 *   -------------------------------------------------------------------------  --------------------------------
 *   cugraph::pagerank(handle, view, weights, nullopt, nullopt, nullopt,          mgb200_cugraph_pagerank_run() with
 *     alpha, epsilon, max_iterations)   mage/cpp/cugraph_module/algorithms/       n_personalization == 0
 *     pagerank.cu:80-91
 *   cugraph::pagerank(..., personalization = (vertices, values), ...)            mgb200_cugraph_pagerank_run() with
 *     mage/cpp/cugraph_module/algorithms/personalized_pagerank.cu:141-152         the seeds
 *
 * The arithmetic is rapidsai/cugraph's (third party, absent from the reference checkout; restated in
 * oracle/cugraph_pagerank_oracle.c and pinned on the reference's e2e fixtures):
 *   pr_0 = 1/N;  p = values / sum(values) on the seeds, 0 elsewhere (no seeds: p = 1/N)
 *   repeat: dangling = sum of pr over vertices without out-edges
 *           new[v] = alpha * sum_{u->v} pr[u] / outdeg(u) + (alpha * dangling + 1 - alpha) * p[v]
 *           stop when sum_v |new[v] - pr[v]| < epsilon (converged) or after max_iterations (not converged)
 * Differences from the in-tree algorithm (mgb200_pagerank.h): dangling mass is redistributed, the stop test is the L1
 * norm, the result is not renormalised.  Edge weights: a handle from mgb200_graph_create_host_weighted_u32() carries one
 * non-negative FP64 weight per edge (new[v] sums w(u,v) * pr[u] / out_w[u], out_w = sum of u's out-edge weights; the
 * modules' weight_property, default weight 1.0); on any other handle every edge counts 1.  Multi-edges count with
 * multiplicity.  The out-weight sums are accumulated with FP64 atomics at build time: weighted results are
 * reproducible to rounding, not bitwise; unweighted ones are bit-reproducible.
 * Single partition only.  No CPU fallback.  Tolerance-based parity (1e-9 relative vs the restatement): cuGraph's own
 * summation order is not reproducible run to run.
 */
#ifndef MGB200_PERSONALIZED_H
#define MGB200_PERSONALIZED_H

#include "mgb200_pagerank.h"

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

typedef struct mgb200_cugraph_params {
  uint64_t max_iterations; /* module default 100 */
  double damping_factor;   /* alpha, module default 0.85 */
  double stop_epsilon;     /* L1 tolerance, module default 1e-5 */
  uint64_t n_personalization;              /* 0: plain PageRank (uniform teleport) */
  const uint64_t *personalization_vertices; /* dense vertex ids < node_count (host memory) */
  const double *personalization_values;     /* host memory; normalised to sum 1; the sum must be > 0 */
} mgb200_cugraph_params;

typedef struct mgb200_cugraph_stats {
  uint64_t iterations;
  int converged;        /* 0: max_iterations ended the loop (cuGraph reports this in its metadata) */
  double last_diff_sum; /* L1 distance of the last two iterates */
  double iterate_ms;    /* CUDA-event time of the loop */
  uint64_t kernel_launches;
} mgb200_cugraph_stats;

/* A single-partition graph handle with edge weights (dense 32-bit ids, host memory).  The in-tree PageRank and Katz on
 * such a handle ignore the weights (their reference algorithms are unweighted). */
int mgb200_graph_create_host_weighted_u32(int device, uint64_t n, uint64_t m, const uint32_t *from, const uint32_t *to,
                                         const double *weight, mgb200_graph **out);

/* rank_out: node_count doubles, HOST memory, original vertex-id order. */
int mgb200_cugraph_pagerank_run(mgb200_graph *g, const mgb200_cugraph_params *params, double *rank_out,
                                mgb200_cugraph_stats *stats);

/* ---- HITS hubs and authorities (what the reference's cugraph.hits.get computes) ----------------------------------
 *
 *   reference call site                                                        replaced by
 *   -------------------------------------------------------------------------  --------------------------------
 *   cugraph::hits(handle, view, hubs, authorities, tolerance, max_iterations,    mgb200_hits_run()
 *     false, normalize, false)   mage/cpp/cugraph_module/algorithms/hits.cu
 *
 * The arithmetic is rapidsai/cugraph's (third party, absent from the reference checkout; restated in
 * oracle/cugraph_hits_oracle.c and pinned on the reference's e2e fixtures mage/tests/e2e/hits_test/test_cugraph_*):
 *   prev = 1/N everywhere
 *   repeat: auth[v] = sum_{u->v} prev[u];  auth /= max(auth)
 *           hubs[u] = sum_{u->v} auth[v];  hubs /= max(hubs)
 *           diff = sum_v |hubs[v] - prev[v]|;  ++iterations
 *           stop when diff < N * tolerance (converged) or iterations >= max_iterations (not converged);  prev = hubs
 *   normalized: hubs /= sum(hubs), auth /= sum(auth)
 * Multi-edges count with multiplicity, self-loops count, edge weights play no part.  N is node_count: a vertex without
 * edges ends with 0 in both vectors but counts in N (the query module passes only the vertices that occur in an edge,
 * as cuGraph's renumbering does).  Two choices the fixtures do not decide:
 *   - after max_iterations without convergence the last iterate is returned with stats.converged = 0 (no error);
 *   - max_iterations = 0 runs one iteration; the module's negative INTEGER wraps through size_t and runs to convergence.
 * A graph with n > 0 and no edges returns all zeros, converged = 1 and 0 iterations.
 * Device side (hits.cu): the graph is built twice from one COO -- the forward handle gathers auth = A^T hubs, the
 * reverse handle (the same COO with the endpoints swapped) gathers hubs = A auth -- with PageRank's layout and gather
 * kernels on each.  Every reduction is two-stage with a fixed tree: results are bit-reproducible run to run and under
 * every gather variant.  Single partition only.  No CPU fallback. */

typedef struct mgb200_hits_graph mgb200_hits_graph; /* forward + reverse handles of one COO, one device */

typedef struct mgb200_hits_params {
  uint64_t max_iterations; /* module default 100 */
  double tolerance;        /* module default 1e-5; the stop test is diff < node_count * tolerance */
  int normalized;          /* module default true: both vectors scaled to sum 1 */
} mgb200_hits_params;

typedef struct mgb200_hits_stats {
  uint64_t iterations;
  int converged;            /* 0: max_iterations ended the loop */
  double last_diff_sum;     /* L1 distance of the last two hub iterates (both max-scaled) */
  double iterate_ms;        /* CUDA-event time of the loop and the output writes */
  uint64_t kernel_launches;
} mgb200_hits_stats;

/* One COO (dense 32-bit ids < n, host memory), both directions built on `device`. */
int mgb200_hits_graph_create_host_u32(int device, uint64_t n, uint64_t m, const uint32_t *from, const uint32_t *to,
                                      mgb200_hits_graph **out);
/* Layout of the forward handle (rows = in-edges: authorities) and of the reverse one (rows = out-edges: hubs). */
int mgb200_hits_graph_get_info(const mgb200_hits_graph *g, mgb200_graph_info *forward, mgb200_graph_info *reverse);
void mgb200_hits_graph_destroy(mgb200_hits_graph *g);
/* hubs_out / authorities_out: node_count doubles each, HOST memory, original vertex-id order. */
int mgb200_hits_run(mgb200_hits_graph *g, const mgb200_hits_params *params, double *hubs_out, double *authorities_out,
                    mgb200_hits_stats *stats);
/* Create + run + destroy on device MGB200_DEVICE (default 0). */
int mgb200_hits(uint64_t n, uint64_t m, const uint32_t *from, const uint32_t *to, const mgb200_hits_params *params,
                double *hubs_out, double *authorities_out, mgb200_hits_stats *stats);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* MGB200_PERSONALIZED_H */

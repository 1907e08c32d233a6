/*
 * oracle/cugraph_hits_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the HITS the reference's cuGraph module calls:
 *   mage/cpp/cugraph_module/algorithms/hits.cu    cugraph::hits(handle, view, hubs, authorities, tolerance,
 *                                                   max_iterations, has_initial_hubs_guess = false, normalize, false)
 * The arithmetic lives in a THIRD-PARTY dependency that is absent from the reference checkout (rapidsai/cugraph).
 * Restated here and pinned on the reference's own e2e fixtures (mage/tests/e2e/hits_test/test_cugraph_*,
 * tests/golden/hits_e2e.json; 4-6 printed digits):
 *     prev = 1/N everywhere;  it = 0
 *     repeat:  auth[v] = sum_{u->v} prev[u];   auth /= max(auth)
 *              hubs[u] = sum_{u->v} auth[v];   hubs /= max(hubs)
 *              diff = sum_v |hubs[v] - prev[v]|;  ++it
 *              stop if diff < N * tolerance (converged) or it >= max_iterations (not converged);  prev = hubs
 *     normalized: hubs /= sum(hubs), auth /= sum(auth)
 * Multi-edges count with multiplicity, self-loops count.  The stop test on N * tolerance is what the 6-digit fixture
 * decides (with diff < tolerance alone test_cugraph_10_nodes_undirected misses by 8e-5).  max_iterations = 0 runs one
 * iteration.  A graph without edges yields zeros, 0 iterations, converged.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static double max_of(const double *v, uint64_t n) {
  double m = 0.0;
  for (uint64_t i = 0; i < n; ++i)
    if (v[i] > m) m = v[i];
  return m;
}

static double sum_of(const double *v, uint64_t n) {
  double s = 0.0;
  for (uint64_t i = 0; i < n; ++i) s += v[i];
  return s;
}

/* 0 ok; 2 out of memory; 3 bad endpoint */
int oracle_cugraph_hits(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, uint64_t max_iterations,
                        double tolerance, int normalized, double *hubs_out, double *auth_out, uint64_t *iterations_out,
                        int *converged_out, double *last_diff_out) {
  if (iterations_out) *iterations_out = 0;
  if (converged_out) *converged_out = 1;
  if (last_diff_out) *last_diff_out = 0.0;
  for (uint64_t e = 0; e < m; ++e)
    if (from[e] >= n || to[e] >= n) return 3;
  if (n == 0) return 0;
  if (m == 0) {
    memset(hubs_out, 0, n * sizeof(double));
    memset(auth_out, 0, n * sizeof(double));
    return 0;
  }
  double *prev = malloc(n * sizeof(double)), *hubs = malloc(n * sizeof(double)), *auth = malloc(n * sizeof(double));
  if (!prev || !hubs || !auth) {
    free(prev);
    free(hubs);
    free(auth);
    return 2;
  }
  for (uint64_t v = 0; v < n; ++v) prev[v] = 1.0 / (double)n;
  uint64_t it = 0;
  int converged = 0;
  double diff = 0.0;
  for (;;) {
    memset(auth, 0, n * sizeof(double));
    for (uint64_t e = 0; e < m; ++e) auth[to[e]] += prev[from[e]];
    const double ma = max_of(auth, n);
    for (uint64_t v = 0; v < n; ++v) auth[v] /= ma;
    memset(hubs, 0, n * sizeof(double));
    for (uint64_t e = 0; e < m; ++e) hubs[from[e]] += auth[to[e]];
    const double mh = max_of(hubs, n);
    for (uint64_t v = 0; v < n; ++v) hubs[v] /= mh;
    diff = 0.0;
    for (uint64_t v = 0; v < n; ++v) diff += fabs(hubs[v] - prev[v]);
    ++it;
    if (diff < (double)n * tolerance) {
      converged = 1;
      break;
    }
    if (it >= max_iterations) break;
    double *t = prev;
    prev = hubs;
    hubs = t;
  }
  if (normalized) {
    const double sh = sum_of(hubs, n), sa = sum_of(auth, n);
    for (uint64_t v = 0; v < n; ++v) {
      hubs[v] /= sh;
      auth[v] /= sa;
    }
  }
  memcpy(hubs_out, hubs, n * sizeof(double));
  memcpy(auth_out, auth, n * sizeof(double));
  if (iterations_out) *iterations_out = it;
  if (converged_out) *converged_out = converged;
  if (last_diff_out) *last_diff_out = diff;
  free(prev);
  free(hubs);
  free(auth);
  return 0;
}

/*
 * oracle/biconnectivity_oracle.c -- CHECKER (test infrastructure, never product code): bridges and biconnected
 * components of the undirected multigraph view, by an iterative (explicit-stack) Hopcroft-Tarjan DFS.  The partition is
 * the one of the reference's bridges.get and biconnected_components.get (mage/cpp/bridges_module,
 * mage/cpp/biconnected_components_module), whose recursive DFS overflows a thread stack on large graphs.
 *
 * Every edge u -> v is in the lists of both u and v and is told apart by its COO position, so a parallel copy of a
 * tree edge is a back edge: a doubled edge is never a bridge, and both copies share a component.  Self-loops are
 * skipped.  Output per COO edge e:
 *   bridge[e] = 1 iff e is a bridge;
 *   bcc[e]    = the number of e's biconnected component, -1 for a self-loop; components are numbered in the order of
 *               their first edge in the COO.
 * Either output may be NULL.  Returns 0 on success, 1 on an endpoint >= n, 2 when memory runs out.
 */
#include <stdint.h>
#include <stdlib.h>

int oracle_biconnectivity(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, uint8_t *bridge_out,
                          int64_t *bcc_out) {
  for (uint64_t e = 0; e < m; ++e)
    if (from[e] >= n || to[e] >= n) return 1;
  uint64_t *ptr = calloc(n + 1, sizeof(uint64_t));
  uint64_t *adj_edge = malloc((2 * m + 1) * sizeof(uint64_t));
  uint64_t *disc = calloc(n + 1, sizeof(uint64_t)); /* 0 = not visited, else 1 + discovery index */
  uint64_t *low = malloc((n + 1) * sizeof(uint64_t));
  uint64_t *cursor = malloc((n + 1) * sizeof(uint64_t));
  uint64_t *parent_edge = malloc((n + 1) * sizeof(uint64_t));
  uint64_t *vstack = malloc((n + 1) * sizeof(uint64_t));
  uint64_t *estack = malloc((m + 1) * sizeof(uint64_t));
  int64_t *label = malloc((m + 1) * sizeof(int64_t));
  int64_t *renumber = malloc((m + 1) * sizeof(int64_t));
  int rc = 0;
  if (!ptr || !adj_edge || !disc || !low || !cursor || !parent_edge || !vstack || !estack || !label || !renumber) {
    rc = 2;
    goto done;
  }
  for (uint64_t e = 0; e < m; ++e) {
    label[e] = -1;
    if (bridge_out) bridge_out[e] = 0;
    if (from[e] == to[e]) continue;
    ptr[from[e] + 1]++;
    ptr[to[e] + 1]++;
  }
  for (uint64_t v = 0; v < n; ++v) ptr[v + 1] += ptr[v];
  for (uint64_t e = 0; e < m; ++e) { /* ptr[v] runs ahead while filling, then is shifted back */
    if (from[e] == to[e]) continue;
    adj_edge[ptr[from[e]]++] = e;
    adj_edge[ptr[to[e]]++] = e;
  }
  for (uint64_t v = n; v > 0; --v) ptr[v] = ptr[v - 1];
  if (n) ptr[0] = 0;

  uint64_t time = 0, components = 0, etop = 0;
  for (uint64_t s = 0; s < n; ++s) {
    if (disc[s]) continue;
    uint64_t vtop = 0;
    vstack[vtop++] = s;
    disc[s] = low[s] = ++time;
    cursor[s] = ptr[s];
    parent_edge[s] = UINT64_MAX;
    while (vtop) {
      const uint64_t v = vstack[vtop - 1];
      if (cursor[v] < ptr[v + 1]) {
        const uint64_t e = adj_edge[cursor[v]++];
        if (e == parent_edge[v]) continue;
        const uint64_t w = from[e] == v ? to[e] : from[e];
        if (!disc[w]) { /* tree edge: descend */
          estack[etop++] = e;
          disc[w] = low[w] = ++time;
          cursor[w] = ptr[w];
          parent_edge[w] = e;
          vstack[vtop++] = w;
        } else if (disc[w] < disc[v]) { /* back edge (or a parallel copy of the tree edge) */
          estack[etop++] = e;
          if (disc[w] < low[v]) low[v] = disc[w];
        } /* else: seen from the descendant w already */
        continue;
      }
      --vtop; /* v is finished: close the tree edge (p, v) */
      if (!vtop) break;
      const uint64_t p = vstack[vtop - 1], pe = parent_edge[v];
      if (low[v] < low[p]) low[p] = low[v];
      if (low[v] > disc[p] && bridge_out) bridge_out[pe] = 1;
      if (low[v] >= disc[p]) { /* p separates v's subtree: pop one component */
        uint64_t e;
        do {
          e = estack[--etop];
          label[e] = (int64_t)components;
        } while (e != pe);
        ++components;
      }
    }
  }
  if (bcc_out) { /* number the components by their first edge */
    for (uint64_t c = 0; c < components; ++c) renumber[c] = -1;
    int64_t next = 0;
    for (uint64_t e = 0; e < m; ++e) {
      if (label[e] < 0) {
        bcc_out[e] = -1;
        continue;
      }
      if (renumber[label[e]] < 0) renumber[label[e]] = next++;
      bcc_out[e] = renumber[label[e]];
    }
  }
done:
  free(ptr);
  free(adj_edge);
  free(disc);
  free(low);
  free(cursor);
  free(parent_edge);
  free(vstack);
  free(estack);
  free(label);
  free(renumber);
  return rc;
}

/*
 * oracle/bipartite_oracle.c -- CHECKER (test infrastructure, never product code): a plain-C restatement of the
 * reference's maximum bipartite matching (mage/cpp/bipartite_matching_module/algorithm/bipartite_matching.cpp).
 *
 * Colouring, the reference's rule: a BFS over the undirected view (every edge u -> v in the lists of both u and v)
 * from every vertex not yet coloured, in dense order; a self-loop, or an edge between two vertices of the same colour,
 * makes the answer 0.  Otherwise the answer is the size of a maximum matching between the two colour classes, found
 * here by Hopcroft-Karp with an iterative DFS (the reference's recursive Kuhn needs a stack as deep as the longest
 * augmenting path).  *matched receives the answer; mate (may be NULL) receives n partners, -1 for an unmatched vertex.
 * Returns 0 on success, 1 on an endpoint >= n, 2 when memory runs out.
 */
#include <stdint.h>
#include <stdlib.h>

#define NONE UINT32_MAX

int oracle_bipartite_matching(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, uint64_t *matched,
                              int64_t *mate_out) {
  *matched = 0;
  for (uint64_t e = 0; e < m; ++e)
    if (from[e] >= n || to[e] >= n) return 1;
  for (uint64_t v = 0; mate_out && v < n; ++v) mate_out[v] = -1;
  if (n == 0) return 0;
  for (uint64_t e = 0; e < m; ++e)
    if (from[e] == to[e]) return 0; /* a self-loop */
  uint64_t *ptr = calloc(n + 1, sizeof(uint64_t));
  uint32_t *adj = malloc((2 * m + 1) * sizeof(uint32_t));
  uint32_t *queue = malloc(n * sizeof(uint32_t));
  int8_t *colour = malloc(n);
  uint32_t *mate = malloc(n * sizeof(uint32_t));
  uint32_t *dist = malloc(n * sizeof(uint32_t));
  uint64_t *it = malloc(n * sizeof(uint64_t));
  uint32_t *stack = malloc(n * sizeof(uint32_t));
  int rc = 0;
  if (!ptr || !adj || !queue || !colour || !mate || !dist || !it || !stack) {
    rc = 2;
    goto done;
  }
  for (uint64_t e = 0; e < m; ++e) {
    ptr[from[e] + 1]++;
    ptr[to[e] + 1]++;
  }
  for (uint64_t v = 0; v < n; ++v) ptr[v + 1] += ptr[v];
  for (uint64_t e = 0; e < m; ++e) { /* ptr[v] runs ahead while filling, then is shifted back */
    adj[ptr[from[e]]++] = (uint32_t)to[e];
    adj[ptr[to[e]]++] = (uint32_t)from[e];
  }
  for (uint64_t v = n; v > 0; --v) ptr[v] = ptr[v - 1];
  ptr[0] = 0;

  /* colouring: 1 for a BFS start, 0 / 1 alternating below it */
  for (uint64_t v = 0; v < n; ++v) colour[v] = -1;
  for (uint64_t s = 0; s < n; ++s) {
    if (colour[s] != -1) continue;
    uint64_t head = 0, tail = 0;
    colour[s] = 1;
    queue[tail++] = (uint32_t)s;
    while (head < tail) {
      const uint32_t u = queue[head++];
      for (uint64_t i = ptr[u]; i < ptr[u + 1]; ++i) {
        const uint32_t w = adj[i];
        if (colour[w] == colour[u]) goto done; /* not bipartite: the answer stays 0 */
        if (colour[w] == -1) {
          colour[w] = (int8_t)(1 - colour[u]);
          queue[tail++] = w;
        }
      }
    }
  }

  /* Hopcroft-Karp from the colour-0 side */
  for (uint64_t v = 0; v < n; ++v) mate[v] = NONE;
  for (;;) {
    uint64_t head = 0, tail = 0;
    int found = 0;
    for (uint64_t u = 0; u < n; ++u) {
      dist[u] = NONE;
      if (colour[u] == 0 && mate[u] == NONE) {
        dist[u] = 0;
        queue[tail++] = (uint32_t)u;
      }
    }
    while (head < tail) { /* layers of left vertices */
      const uint32_t u = queue[head++];
      for (uint64_t i = ptr[u]; i < ptr[u + 1]; ++i) {
        const uint32_t x = mate[adj[i]];
        if (x == NONE) found = 1;
        else if (dist[x] == NONE) {
          dist[x] = dist[u] + 1;
          queue[tail++] = x;
        }
      }
    }
    if (!found) break;
    for (uint64_t v = 0; v < n; ++v) it[v] = ptr[v];
    for (uint64_t s = 0; s < n; ++s) {
      if (colour[s] != 0 || mate[s] != NONE) continue;
      uint64_t top = 0;
      stack[top++] = (uint32_t)s;
      while (top > 0) {
        const uint32_t u = stack[top - 1];
        if (it[u] == ptr[u + 1]) {
          dist[u] = NONE; /* a dead end for the rest of the phase */
          --top;
          continue;
        }
        const uint32_t w = adj[it[u]++];
        const uint32_t x = mate[w];
        if (x == NONE) { /* augment: the right vertex of every level is the entry just read */
          for (uint64_t k = 0; k < top; ++k) {
            const uint32_t l = stack[k], r = adj[it[l] - 1];
            mate[l] = r;
            mate[r] = l;
          }
          ++*matched;
          break;
        }
        if (dist[x] == dist[u] + 1) stack[top++] = x;
      }
    }
  }
  for (uint64_t v = 0; mate_out && v < n; ++v) mate_out[v] = mate[v] == NONE ? -1 : (int64_t)mate[v];
done:
  free(ptr);
  free(adj);
  free(queue);
  free(colour);
  free(mate);
  free(dist);
  free(it);
  free(stack);
  return rc;
}

/*
 * oracle/wcc_oracle.c -- CHECKER (test infrastructure, never product code): a plain-C restatement of the reference's
 * weakly connected components (mage/cpp/connectivity_module/connectivity_module.cpp:41-84).
 *
 * The undirected view holds every edge u -> v in the lists of both u and v.  A BFS starts from every vertex not yet
 * reached, in dense order, and gives all it reaches the next component number.  Self-loops and multi-edges change
 * nothing.  Returns 0 on success, 1 on an endpoint >= n, 2 when memory runs out.
 */
#include <stdint.h>
#include <stdlib.h>

int oracle_wcc(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, int64_t *component) {
  for (uint64_t e = 0; e < m; ++e)
    if (from[e] >= n || to[e] >= n) return 1;
  if (n == 0) return 0;
  uint64_t *ptr = calloc(n + 1, sizeof(uint64_t));
  uint32_t *adj = malloc((2 * m + 1) * sizeof(uint32_t));
  uint32_t *queue = malloc(n * sizeof(uint32_t));
  if (!ptr || !adj || !queue) {
    free(ptr);
    free(adj);
    free(queue);
    return 2;
  }
  for (uint64_t e = 0; e < m; ++e) {
    ptr[from[e] + 1]++;
    ptr[to[e] + 1]++;
  }
  for (uint64_t v = 0; v < n; ++v) ptr[v + 1] += ptr[v];
  for (uint64_t e = 0; e < m; ++e) {  /* ptr[v] runs ahead while filling, then is shifted back */
    adj[ptr[from[e]]++] = (uint32_t)to[e];
    adj[ptr[to[e]]++] = (uint32_t)from[e];
  }
  for (uint64_t v = n; v > 0; --v) ptr[v] = ptr[v - 1];
  ptr[0] = 0;
  for (uint64_t v = 0; v < n; ++v) component[v] = -1;
  int64_t next = 0;
  for (uint64_t s = 0; s < n; ++s) {
    if (component[s] >= 0) continue;
    uint64_t head = 0, tail = 0;
    queue[tail++] = (uint32_t)s;
    component[s] = next;
    while (head < tail) {
      const uint32_t v = queue[head++];
      for (uint64_t k = ptr[v]; k < ptr[v + 1]; ++k) {
        const uint32_t w = adj[k];
        if (component[w] >= 0) continue;
        component[w] = next;
        queue[tail++] = w;
      }
    }
    ++next;
  }
  free(ptr);
  free(adj);
  free(queue);
  return 0;
}

/*
 * oracle/scc_oracle.c -- CHECKER (test infrastructure, never product code): strongly connected components, the
 * partition networkx.strongly_connected_components gives on the MultiDiGraph of all vertices and edges (the reference's
 * nxalg.strongly_connected_components), by Tarjan's algorithm.
 *
 * The depth-first search keeps its own stack (vertex, next out-entry) instead of recursing: the search into a giant
 * component can be nearly n deep.  component[v] is numbered in the order of each component's smallest vertex id, the
 * numbering of mgb200_scc_run.  Self-loops and multi-edges change nothing.  Returns 0 on success, 1 on an endpoint
 * >= n, 2 when memory runs out.
 */
#include <stdint.h>
#include <stdlib.h>

int oracle_scc(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, int64_t *component) {
  for (uint64_t e = 0; e < m; ++e)
    if (from[e] >= n || to[e] >= n) return 1;
  if (n == 0) return 0;
  uint64_t *ptr = calloc(n + 1, sizeof(uint64_t));
  uint32_t *adj = malloc((m + 1) * sizeof(uint32_t));
  uint64_t *index = malloc(n * sizeof(uint64_t));   /* discovery order + 1, 0 = not yet discovered */
  uint64_t *low = malloc(n * sizeof(uint64_t));
  uint64_t *edge = malloc(n * sizeof(uint64_t));    /* the call stack: next out-entry of each vertex on it */
  uint32_t *call = malloc(n * sizeof(uint32_t));
  uint32_t *stack = malloc(n * sizeof(uint32_t));   /* Tarjan's stack */
  uint32_t *smallest = malloc(n * sizeof(uint32_t)); /* per component found: its smallest vertex */
  uint8_t *on_stack = calloc(n, 1);
  if (!ptr || !adj || !index || !low || !edge || !call || !stack || !smallest || !on_stack) {
    free(ptr), free(adj), free(index), free(low), free(edge), free(call), free(stack), free(smallest), free(on_stack);
    return 2;
  }
  for (uint64_t e = 0; e < m; ++e) ptr[from[e] + 1]++;
  for (uint64_t v = 0; v < n; ++v) ptr[v + 1] += ptr[v];
  for (uint64_t e = 0; e < m; ++e) adj[ptr[from[e]]++] = (uint32_t)to[e];
  for (uint64_t v = n; v > 0; --v) ptr[v] = ptr[v - 1];
  ptr[0] = 0;
  for (uint64_t v = 0; v < n; ++v) index[v] = 0, component[v] = -1;

  uint64_t counter = 0, top = 0, found = 0;
  for (uint64_t s = 0; s < n; ++s) {
    if (index[s]) continue;
    uint64_t depth = 0;
    call[depth++] = (uint32_t)s;
    index[s] = low[s] = ++counter;
    edge[s] = ptr[s];
    stack[top++] = (uint32_t)s;
    on_stack[s] = 1;
    while (depth) {
      const uint32_t v = call[depth - 1];
      if (edge[v] < ptr[v + 1]) {
        const uint32_t w = adj[edge[v]++];
        if (!index[w]) {
          index[w] = low[w] = ++counter;
          edge[w] = ptr[w];
          stack[top++] = w;
          on_stack[w] = 1;
          call[depth++] = w;
        } else if (on_stack[w] && index[w] < low[v]) {
          low[v] = index[w];
        }
        continue;
      }
      --depth;  /* v is done: it closes a component if nothing on the stack above it reaches lower */
      if (depth && low[v] < low[call[depth - 1]]) low[call[depth - 1]] = low[v];
      if (low[v] != index[v]) continue;
      uint32_t least = v, w;
      uint64_t base = top;
      do {
        w = stack[--base];
        if (w < least) least = w;
      } while (w != v);
      for (uint64_t i = base; i < top; ++i) {
        on_stack[stack[i]] = 0;
        component[stack[i]] = (int64_t)found;  /* provisional: the order components were closed */
      }
      smallest[found++] = least;
      top = base;
    }
  }
  /* renumber: rank of each component's smallest vertex among all components' smallest vertices */
  int64_t *rank = (int64_t *)low;  /* low is no longer needed; reuse it as component -> final number */
  for (uint64_t c = 0; c < found; ++c) rank[c] = -1;
  int64_t next = 0;
  for (uint64_t v = 0; v < n; ++v) {
    const int64_t c = component[v];
    if (smallest[c] == v) rank[c] = next++;
  }
  for (uint64_t v = 0; v < n; ++v) component[v] = rank[component[v]];
  free(ptr), free(adj), free(index), free(low), free(edge), free(call), free(stack), free(smallest), free(on_stack);
  return 0;
}

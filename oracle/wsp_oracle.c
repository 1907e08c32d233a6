/*
 * oracle/wsp_oracle.c -- CHECKER (test infrastructure, never product code): a plain-C restatement of the reference's
 * weighted shortest path expansion, ExpandWeightedShortestPathCursor (src/query/plan/operator.cpp:2917-3267), for one
 * source, an unbound target, one numeric edge property as the weight and no filter lambda.
 *
 * Step by step, as the cursor does it:
 *   - a binary min-heap of (weight, depth, vertex); the source enters with depth 0 and a Null total, which behaves as
 *     +0.0 here (the first hop's total is w_1 itself, :2961, and fl(+0 + w) = w for w >= +0);
 *   - the state key is (v, bounded ? depth : 0) (:2998);
 *   - a popped state already in total_cost is skipped; otherwise its cost is recorded and, while depth < upper_bound,
 *     every walked-direction entry of v is evaluated (out-list first, then in-list for BOTH, :3056-3087).  The prune of
 *     :3039 looks up the state (neighbour, depth of the EXPANDED vertex) and drops the push when that state's cost is
 *     <= the new total; otherwise (new total, depth + 1, neighbour) is pushed;
 *   - a vertex is yielded at its first popped state (:3160); the source never is (:3135).
 * Ties in the heap go to the smaller depth, then the smaller vertex id: that is one of the orders the reference's
 * priority queue may pop in, so cursor_depth is one valid size(le).
 *
 * An evaluated entry whose weight is NaN or negative makes the reference raise (:2919-2942).  Here the entry is skipped
 * instead and the smallest COO index among the evaluated invalid entries is reported, which is the same error /
 * no-error outcome.  Weights -0.0 count as +0.0.
 *
 * Canonical hops (the fewest edges among the paths the reference can return):
 *   unbounded  the BFS depth of v over tight entries (d[v] == fl(d[u] + w));
 *   bounded    the smallest k with d_k[v] == d_u[v], d_k the minimum over walks of at most k edges (Jacobi rounds).
 *
 * Returns 0 on success, 1 on a bad argument (endpoint or source >= n), 2 when memory runs out, 3 when an evaluated
 * weight is invalid (*invalid_edge set), 4 when upper_bound < 1.  dist / cursor_depth / hops get NaN / -1 / -1 for
 * vertices that are not yielded.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  double w;
  int64_t depth;
  uint32_t v;
} Entry;

typedef struct {
  Entry *a;
  uint64_t size, cap;
} Heap;

static int less(const Entry *x, const Entry *y) {
  if (x->w != y->w) return x->w < y->w;
  if (x->depth != y->depth) return x->depth < y->depth;
  return x->v < y->v;
}

static int heap_push(Heap *h, Entry e) {
  if (h->size == h->cap) {
    uint64_t cap = h->cap ? 2 * h->cap : 1024;
    Entry *a = realloc(h->a, cap * sizeof(Entry));
    if (!a) return 0;
    h->a = a;
    h->cap = cap;
  }
  uint64_t i = h->size++;
  while (i > 0) {
    uint64_t p = (i - 1) / 2;
    if (!less(&e, &h->a[p])) break;
    h->a[i] = h->a[p];
    i = p;
  }
  h->a[i] = e;
  return 1;
}

static Entry heap_pop(Heap *h) {
  Entry top = h->a[0], last = h->a[--h->size];
  uint64_t i = 0;
  for (;;) {
    uint64_t c = 2 * i + 1;
    if (c >= h->size) break;
    if (c + 1 < h->size && less(&h->a[c + 1], &h->a[c])) ++c;
    if (!less(&h->a[c], &last)) break;
    h->a[i] = h->a[c];
    i = c;
  }
  if (h->size) h->a[i] = last;
  return top;
}

/* total_cost: state (vertex, depth) -> cost, open addressing */
typedef struct {
  uint64_t *key; /* (depth << 32 | vertex) + 1, 0 = empty */
  double *cost;
  uint64_t cap, size;
} CostMap;

static uint64_t mix(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

static double *map_find(const CostMap *m, uint64_t k) {
  for (uint64_t i = mix(k) & (m->cap - 1);; i = (i + 1) & (m->cap - 1)) {
    if (m->key[i] == 0) return NULL;
    if (m->key[i] == k) return &m->cost[i];
  }
}

static int map_put(CostMap *m, uint64_t k, double c) {
  if (2 * (m->size + 1) > m->cap) {
    CostMap g = {calloc(2 * m->cap, sizeof(uint64_t)), malloc(2 * m->cap * sizeof(double)), 2 * m->cap, 0};
    if (!g.key || !g.cost) {
      free(g.key);
      free(g.cost);
      return 0;
    }
    for (uint64_t i = 0; i < m->cap; ++i)
      if (m->key[i]) map_put(&g, m->key[i], m->cost[i]);
    free(m->key);
    free(m->cost);
    *m = g;
  }
  uint64_t i = mix(k) & (m->cap - 1);
  while (m->key[i] != 0 && m->key[i] != k) i = (i + 1) & (m->cap - 1);
  if (m->key[i] == 0) m->size++;
  m->key[i] = k;
  m->cost[i] = c;
  return 1;
}

static int invalid_weight(double w) { return isnan(w) || w < 0.0; }

int oracle_wsp(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, const double *weight,
               uint64_t source, int direction, int64_t upper_bound, double *dist, int32_t *cursor_depth,
               int32_t *hops, uint64_t *invalid_edge) {
  if (upper_bound < 1) return 4;
  if (source >= n || direction < 0 || direction > 2) return 1;
  for (uint64_t e = 0; e < m; ++e)
    if (from[e] >= n || to[e] >= n) return 1;
  const int bounded = upper_bound != INT64_MAX;
  /* walked lists: entry = COO index; OUT lists by `from`, IN lists by `to`, each in COO order */
  uint64_t *optr = calloc(n + 1, sizeof(uint64_t)), *iptr = calloc(n + 1, sizeof(uint64_t));
  uint64_t *oadj = malloc((m + 1) * sizeof(uint64_t)), *iadj = malloc((m + 1) * sizeof(uint64_t));
  double *d = malloc(n * sizeof(double));
  char *yielded = calloc(n, 1);
  uint32_t *queue = malloc(n * sizeof(uint32_t));
  double *prev = malloc(n * sizeof(double));
  CostMap cost = {calloc(1024, sizeof(uint64_t)), malloc(1024 * sizeof(double)), 1024, 0};
  Heap heap = {NULL, 0, 0};
  int rc = 0;
  uint64_t invalid = UINT64_MAX;
  if (!optr || !iptr || !oadj || !iadj || !d || !yielded || !queue || !prev || !cost.key || !cost.cost) {
    rc = 2;
    goto done;
  }
  for (uint64_t e = 0; e < m; ++e) {
    optr[from[e] + 1]++;
    iptr[to[e] + 1]++;
  }
  for (uint64_t v = 0; v < n; ++v) {
    optr[v + 1] += optr[v];
    iptr[v + 1] += iptr[v];
  }
  for (uint64_t e = 0; e < m; ++e) {
    oadj[optr[from[e]]++] = e;
    iadj[iptr[to[e]]++] = e;
  }
  for (uint64_t v = n; v > 0; --v) {
    optr[v] = optr[v - 1];
    iptr[v] = iptr[v - 1];
  }
  optr[0] = iptr[0] = 0;
  for (uint64_t v = 0; v < n; ++v) {
    d[v] = NAN;
    dist[v] = NAN;
    cursor_depth[v] = -1;
    hops[v] = -1;
  }

  /* ---- the cursor ---- */
  yielded[source] = 1;
  if (!heap_push(&heap, (Entry){0.0, 0, (uint32_t)source})) {
    rc = 2;
    goto done;
  }
  while (heap.size) {
    const Entry top = heap_pop(&heap);
    if (bounded) {
      const uint64_t key = (((uint64_t)top.depth << 32) | top.v) + 1;
      if (map_find(&cost, key)) continue;
      if (!map_put(&cost, key, top.w)) {
        rc = 2;
        goto done;
      }
    } else {  /* state (v, 0): a plain array (d[] holds the processed cost, NaN = not processed) */
      if (!isnan(d[top.v])) continue;
      d[top.v] = top.w;
    }
    if (top.depth < upper_bound) {
      for (int side = 0; side < 2; ++side) {
        if ((side == 0 && direction == 1) || (side == 1 && direction == 0)) continue;
        const uint64_t *ptr = side == 0 ? optr : iptr, *adj = side == 0 ? oadj : iadj;
        for (uint64_t k = ptr[top.v]; k < ptr[top.v + 1]; ++k) {
          const uint64_t e = adj[k];
          const uint32_t x = (uint32_t)(side == 0 ? to[e] : from[e]);
          double w = weight[e];
          if (invalid_weight(w)) {
            if (e < invalid) invalid = e;
            continue;
          }
          if (w == 0.0) w = 0.0;
          const double next = top.w + w;
          const double *found = bounded ? map_find(&cost, (((uint64_t)top.depth << 32) | x) + 1)
                                        : (isnan(d[x]) ? NULL : &d[x]);
          if (found && *found <= next) continue;
          if (!heap_push(&heap, (Entry){next, top.depth + 1, x})) {
            rc = 2;
            goto done;
          }
        }
      }
    }
    if (yielded[top.v]) continue;
    yielded[top.v] = 1;
    dist[top.v] = top.w;
    cursor_depth[top.v] = (int32_t)top.depth;
  }

  /* ---- canonical hops ---- */
  if (!bounded) {
    for (uint64_t v = 0; v < n; ++v) d[v] = dist[v];
    d[source] = 0.0;
    hops[source] = 0;
    uint64_t head = 0, tail = 0;
    queue[tail++] = (uint32_t)source;
    while (head < tail) {
      const uint32_t u = queue[head++];
      for (int side = 0; side < 2; ++side) {
        if ((side == 0 && direction == 1) || (side == 1 && direction == 0)) continue;
        const uint64_t *ptr = side == 0 ? optr : iptr, *adj = side == 0 ? oadj : iadj;
        for (uint64_t k = ptr[u]; k < ptr[u + 1]; ++k) {
          const uint64_t e = adj[k];
          const uint32_t x = (uint32_t)(side == 0 ? to[e] : from[e]);
          double w = weight[e];
          if (invalid_weight(w) || hops[x] >= 0) continue;
          if (w == 0.0) w = 0.0;
          if (d[u] + w == d[x]) {
            hops[x] = hops[u] + 1;
            queue[tail++] = x;
          }
        }
      }
    }
  } else {
    /* Jacobi rounds: round k reads only d_{k-1} (prev); hops = the round of the last strict improvement */
    for (uint64_t v = 0; v < n; ++v) d[v] = INFINITY, hops[v] = -1;
    char *reached = yielded; /* reuse: reached[v] = d_k[v] is defined */
    memset(reached, 0, n);
    d[source] = 0.0;
    reached[source] = 1;
    hops[source] = 0;
    for (int64_t k = 1; k <= upper_bound; ++k) {
      memcpy(prev, d, n * sizeof(double));
      char *was = malloc(n);
      if (!was) {
        rc = 2;
        goto done;
      }
      memcpy(was, reached, n);
      int changed = 0;
      for (uint64_t e = 0; e < m; ++e) {
        double w = weight[e];
        if (invalid_weight(w)) continue;
        if (w == 0.0) w = 0.0;
        for (int side = 0; side < 2; ++side) {
          if ((side == 0 && direction == 1) || (side == 1 && direction == 0)) continue;
          const uint64_t u = side == 0 ? from[e] : to[e], x = side == 0 ? to[e] : from[e];
          if (!was[u]) continue;
          const double c = prev[u] + w;
          if (!reached[x] || c < d[x]) {
            d[x] = c;
            reached[x] = 1;
            hops[x] = (int32_t)k;
            changed = 1;
          }
        }
      }
      free(was);
      if (!changed) break;
    }
  }
  for (uint64_t v = 0; v < n; ++v)
    if (cursor_depth[v] < 0) hops[v] = -1;
  if (invalid != UINT64_MAX) rc = 3;

done:
  if (invalid_edge) *invalid_edge = invalid;
  free(optr);
  free(iptr);
  free(oadj);
  free(iadj);
  free(d);
  free(yielded);
  free(queue);
  free(prev);
  free(cost.key);
  free(cost.cost);
  free(heap.a);
  return rc;
}

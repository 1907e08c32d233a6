/*
 * mgb200_bfs.h -- C ABI of the GPU-native breadth-first expansion (the NEXT path after PageRank, SURVEY 8f-2 /
 * BASELINE config #5: "BFS expand on RMAT scale-24, one GPU, distances bit-exact vs the reference").
 *
 * Replaces the arithmetic of the reference's engine operator for `MATCH (a)-[*BFS lower..upper]->(b)` with an
 * unbound target -- SingleSourceShortestPathCursor, src/query/plan/operator.cpp:2692-2912: level-synchronous
 * expansion from one source, visited-on-discovery, direction OUT / IN / BOTH, depth bounds (default 1..inf),
 * the source itself is never produced.  The operator lives inside the engine (no plugin boundary exists for it),
 * so this ABI is what a new read procedure (e.g. gpu_bfs.distances(source)) would call; see INTEGRATION.md.
 *
 * Output: dist[v] = the BFS depth at which the reference emits v, or -1 when it does not (unreachable, the
 * source, or depth outside [lower_bound, upper_bound]).  Integer work: parity is bit-exact.
 */
#ifndef MGB200_BFS_H
#define MGB200_BFS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

#define MGB200_BFS_OUT 0  /* EdgeAtom::Direction::OUT  */
#define MGB200_BFS_IN 1   /* EdgeAtom::Direction::IN   */
#define MGB200_BFS_BOTH 2 /* EdgeAtom::Direction::BOTH */

typedef struct mgb200_bfs_graph mgb200_bfs_graph; /* device-resident CSR (out) + CSC (in); also walked by mgb200_bc_run */

typedef struct mgb200_bfs_stats {
  uint32_t levels;            /* depth of the deepest discovered vertex                                   */
  uint32_t top_down_levels;   /* levels expanded frontier-first (queue, atomicCAS on the depth array)     */
  uint32_t bottom_up_levels;  /* levels expanded by the unvisited vertices looking for a frontier parent  */
  uint64_t reached;           /* vertices discovered (source excluded), before the bounds filter          */
  uint64_t edges_inspected;   /* adjacency entries actually read                                          */
  double traverse_ms;         /* CUDA-event time of the expansion (depth array initialised .. last level) */
  uint64_t kernel_launches;
} mgb200_bfs_stats;

/* COO on the device (uint32 endpoints < n, read not consumed) -> CSR + CSC, both sorted. */
int mgb200_bfs_graph_create_device(int device, uint64_t n, uint64_t m, const uint32_t *d_from, const uint32_t *d_to,
                                   mgb200_bfs_graph **out);
/* COO in host memory (uint64 endpoints). */
int mgb200_bfs_graph_create_host(int device, uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                 mgb200_bfs_graph **out);
void mgb200_bfs_graph_destroy(mgb200_bfs_graph *g);

/* lower_bound / upper_bound: pass 1 and INT64_MAX for the reference's defaults (operator.cpp:2824-2828).
 * dist_out: n int32 values, host memory (dist_on_device = 0) or memory of the graph's device (1). */
int mgb200_bfs_run(mgb200_bfs_graph *g, uint64_t source, int direction, int64_t lower_bound, int64_t upper_bound,
                   int32_t *dist_out, int dist_on_device, mgb200_bfs_stats *stats);

/*
 * Exact betweenness centrality (Brandes) on the same device graph: the arithmetic of the reference's
 * betweenness_centrality_alg::BetweennessCentrality (mage/cpp/betweenness_centrality_module/algorithm/
 * betweenness_centrality.cpp:24-146).  One level-synchronous BFS per source counts shortest paths sigma as
 * uint64_t, wrapping modulo 2^64 like the reference; a backward sweep accumulates the dependencies delta; every
 * vertex c != s gains delta[c] (directed) or delta[c] / 2 (undirected).  directed = 0 walks the undirected view
 * (out- and in-lists together, multi-edges with their multiplicity); self-loops have no effect.
 * Sources are processed in batches of MGB200_BC_BATCH, summed into each vertex in ascending source order, so two
 * runs are bit-identical.  Without a device every call fails with MGB200_ERR_CUDA.
 */
#define MGB200_BC_BATCH 32 /* sources per batch: one warp lane each */

typedef struct mgb200_bc_stats {
  uint64_t sources;          /* source_end - source_begin                                        */
  uint64_t batches;          /* batches of up to MGB200_BC_BATCH sources                          */
  uint32_t batch_width;      /* MGB200_BC_BATCH                                                   */
  uint32_t max_levels;       /* deepest BFS level reached by any source                           */
  uint64_t edges_traversed;  /* adjacency entries read, forward and backward sweeps together      */
  double run_ms;             /* CUDA-event time of all batches (state initialisation .. last sum) */
  uint64_t kernel_launches;
} mgb200_bc_stats;

/* Un-normalised betweenness summed over the sources [source_begin, source_end) (0 <= begin <= end <= n).
 * bc_out: n doubles, host memory (bc_on_device = 0) or memory of the graph's device (1); overwritten, not added to.
 * should_abort (may be NULL) is polled between batches; when it returns non-zero the call returns
 * MGB200_ERR_ABORTED and bc_out is left untouched. */
int mgb200_bc_run(mgb200_bfs_graph *g, int directed, uint64_t source_begin, uint64_t source_end,
                  int (*should_abort)(void *user), void *abort_user, double *bc_out, int bc_on_device,
                  mgb200_bc_stats *stats);

/* The reference function end to end, on device 0: host COO (uint64 endpoints < n) -> bc_out[n] in host memory,
 * all sources, normalised when `normalized` != 0 by (directed ? 1 : 2) / ((n - 1) * (n - 2)) for n > 2. */
int mgb200_betweenness_centrality(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, int directed,
                                  int normalized, double *bc_out);

/*
 * Weakly connected components on the same device graph: the result of the reference's weakly_connected_components.get
 * (mage/cpp/connectivity_module/connectivity_module.cpp:41-84), a BFS over the undirected view (out- and in-lists
 * together) from every unvisited vertex in dense order.  component_out[v] is the number of v's component; components
 * are numbered in the order of their smallest vertex id.  Self-loops and multi-edges change nothing.  The work is
 * integer union-find whose roots are the components' smallest ids, so two runs are byte-identical.  Without a device
 * every call fails with MGB200_ERR_CUDA.
 */
typedef struct mgb200_wcc_stats {
  uint64_t components;         /* number of components                                    */
  uint64_t largest_component;  /* vertices in the largest one                             */
  uint64_t skipped_vertices;   /* vertices whose remaining lists the finish phase skipped */
  uint64_t edges_inspected;    /* adjacency entries read, sampling and finish together    */
  double run_ms;               /* CUDA-event time, parent init .. last label written      */
  uint64_t kernel_launches;
} mgb200_wcc_stats;

/* component_out: n int64 values in host memory.  n == 0 returns MGB200_OK with zero components. */
int mgb200_wcc_run(mgb200_bfs_graph *g, int64_t *component_out, mgb200_wcc_stats *stats);

/* The reference procedure's arithmetic end to end, on device 0: host COO (uint64 endpoints < n) -> component_out[n]. */
int mgb200_weakly_connected_components(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                       int64_t *component_out);

/*
 * Bridges and biconnected components of the undirected multigraph view (every edge in both endpoints' lists), the
 * partition of the reference's bridges.get and biconnected_components.get (mage/cpp/bridges_module,
 * mage/cpp/biconnected_components_module).  Tarjan-Vishkin on a breadth-first spanning forest rooted at each
 * component's smallest id; all integer work, so two runs are byte-identical.  Per edge e of the COO the graph was built
 * from, in the same order:
 *   bridge_out[e] = 1 iff removing e disconnects its endpoints (a doubled edge is never a bridge, a self-loop never is);
 *   bcc_out[e]    = the number of e's biconnected component, -1 for a self-loop.  Components are numbered in the order
 *                   of their first edge in the COO, so the numbering depends neither on thread order nor on the tree.
 * Without a device every call fails with MGB200_ERR_CUDA.
 */
typedef struct mgb200_biconnectivity_stats {
  uint64_t trees;            /* spanning trees with at least one edge                              */
  uint32_t forest_depth;     /* deepest BFS level of the forest (0 when no vertex has a parent)    */
  uint64_t bridges;          /* edges with bridge_out = 1                                          */
  uint64_t components;       /* biconnected components (self-loops belong to none)                 */
  uint64_t edges_inspected;  /* adjacency entries read, forest and low / high passes together      */
  double run_ms;             /* CUDA-event time, first kernel .. last label written (no transfers) */
  uint64_t kernel_launches;
} mgb200_biconnectivity_stats;

/* from / to: the host uint64 COO the graph was built from, in the same order (m must equal the graph's edge count).
 * bridge_out: m uint8 values, bcc_out: m int64 values, both host memory; either may be NULL. */
int mgb200_biconnectivity_run(mgb200_bfs_graph *g, uint64_t m, const uint64_t *from, const uint64_t *to,
                              uint8_t *bridge_out, int64_t *bcc_out, mgb200_biconnectivity_stats *stats);

/* One shot on device 0: host COO (uint64 endpoints < n) -> bridge_out[m] / bcc_out[m] in host memory. */
int mgb200_bridges(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, uint8_t *bridge_out);
int mgb200_biconnected_components(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to, int64_t *bcc_out);

/*
 * Weighted shortest paths from one source on the same device graph: the totals of the reference's
 * `MATCH (a)-[*WSHORTEST ..u (e, n | e.w) total_weight]->(b)` with an unbound target and one numeric edge property as
 * the weight (ExpandWeightedShortestPathCursor, src/query/plan/operator.cpp:2917-3267).
 *
 * Weights are doubles w >= +0 (+inf allowed; -0.0 is stored as +0.0).  A negative or NaN weight is an INVALID entry:
 * it is stored as the quiet NaN 0x7FF8000000000000 | e, where e is the entry's index in the COO given to
 * mgb200_bfs_graph_set_weights (e < 2^51).  Totals are left folds of IEEE round-to-nearest additions; because
 * fl(a + w) is monotone in a and never below a, every relaxation order reaches the same least fixed point, so dist is
 * bit-exact.  upper_bound == INT64_MAX is unbounded (delta-stepping); otherwise at most upper_bound Jacobi Bellman-Ford
 * rounds give the minimum over walks of at most upper_bound edges.  The environment variable MGB200_WSP_DELTA, read at
 * every unbounded call, sets the bucket width when it is a finite number > 0; the width changes the work, not dist.
 *
 * Output per vertex v (host memory):
 *   dist_out[v] = v's total_weight (may be +inf), NaN when v is not produced (unreached, or the source itself);
 *   hops_out[v] = the fewest edges among the paths the reference can return for v, -1 when v is not produced:
 *                 unbounded, the BFS depth of v over tight entries (d[v] == fl(d[u] + w)); bounded, the smallest k with
 *                 d_k[v] == d_upper_bound[v].
 * If an entry the reference would evaluate (an entry of the walked direction out of a vertex that gets expanded) is
 * invalid, the call returns MGB200_ERR_INVALID_WEIGHT and stats->invalid_edge holds the smallest COO index among the
 * evaluated invalid entries; dist_out / hops_out are then unspecified.  Without a device every call fails with
 * MGB200_ERR_CUDA.
 */
#define MGB200_ERR_INVALID_WEIGHT 17 /* an evaluated edge weight is negative or not a number */
#define MGB200_WSP_UNBOUNDED INT64_MAX
#define MGB200_WSP_INVALID_TAG 0x7FF8000000000000ull /* invalid entry = this | COO index */

typedef struct mgb200_wsp_stats {
  uint64_t rounds;             /* relaxation passes: Bellman-Ford rounds, or near-pile passes of all buckets      */
  uint64_t buckets;            /* distance buckets processed (unbounded), 0 when bounded                          */
  uint32_t hop_levels;         /* deepest hops value of a produced vertex                                         */
  double delta;                /* bucket width (unbounded), 0 when bounded                                        */
  uint64_t reached;            /* vertices produced                                                               */
  uint64_t relaxations;        /* (pass, vertex) pairs whose distance a pass lowered                              */
  uint64_t entries_inspected;  /* adjacency entries read, distance passes and the tight-entry BFS together        */
  uint64_t invalid_edge;       /* smallest COO index of an evaluated invalid entry, UINT64_MAX when there is none */
  double run_ms;               /* CUDA-event time, distance init .. last output written (no transfers)            */
  uint64_t kernel_launches;
} mgb200_wsp_stats;

/* Weights of the COO the graph was built from (from / to / weight host arrays of m entries, m equal to the graph's
 * edge count, same pairs in any order).  Builds out_w / in_w aligned with the sorted out- and in-lists; calling it
 * again replaces them.  Duplicates of one (u, v) pair may take each other's weights: no answer depends on that.
 * A COO whose (from, to) pairs differ from the graph's is refused with MGB200_ERR_INVALID_ARGUMENT.  Any failure
 * leaves the graph without weights (never with a mix of the old and the new ones).  Device staging: 24 B per edge
 * plus the sort's temporary, on top of the 16 B per edge the two weight arrays keep. */
int mgb200_bfs_graph_set_weights(mgb200_bfs_graph *g, uint64_t m, const uint64_t *from, const uint64_t *to,
                                 const double *weight);

/* should_abort (may be NULL) is polled between host round trips; non-zero -> MGB200_ERR_ABORTED.  stats may be NULL.
 * upper_bound < 1 -> MGB200_ERR_INVALID_ARGUMENT.  Two runs give byte-identical outputs and stats (run_ms aside). */
int mgb200_wsp_run(mgb200_bfs_graph *g, uint64_t source, int direction, int64_t upper_bound,
                   int (*should_abort)(void *user), void *abort_user, double *dist_out, int32_t *hops_out,
                   mgb200_wsp_stats *stats);

/* One shot on device 0: host COO with weights -> dist_out[n] / hops_out[n] in host memory. */
int mgb200_weighted_shortest_paths(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                   const double *weight, uint64_t source, int direction, int64_t upper_bound,
                                   double *dist_out, int32_t *hops_out);

/*
 * Maximum bipartite matching of the undirected multigraph view on the same device graph: the answer of the reference's
 * bipartite_matching.max (mage/cpp/bipartite_matching_module).  A breadth-first forest from each component's smallest
 * id colours the graph; a self-loop or an edge between two vertices of the same forest level (an odd cycle) means the
 * graph is not bipartite and the answer is 0.  Otherwise the even-depth vertices are the left side, and greedy rounds
 * followed by alternating breadth-first searches from every free left vertex (one phase per search, paths flipped in
 * parallel) grow the matching until a search finds no augmenting path.  Every choice is a minimum over vertex ids, so
 * two runs give byte-identical outputs and stats (run_ms aside).  Without a device every call fails with
 * MGB200_ERR_CUDA.
 */
typedef struct mgb200_matching_stats {
  int bipartite;              /* 0: a self-loop or an odd cycle; nothing matched                  */
  uint64_t left_vertices;     /* even forest depth: the side the searches start from (0 if not bipartite) */
  uint64_t matched;           /* pairs = the reference procedure's answer                          */
  uint64_t initial_matched;   /* pairs after the greedy rounds                                     */
  uint64_t phases;            /* alternating searches, the last one fruitless                      */
  uint32_t max_levels;        /* deepest search level of any phase                                 */
  uint64_t edges_inspected;   /* adjacency entries read: colouring, greedy and searches together   */
  double run_ms;              /* CUDA-event time, first kernel .. last output (no transfers)        */
  uint64_t kernel_launches;
} mgb200_matching_stats;

/* mate_out: n int64 (partner id or -1); cover_out: n uint8 (a minimum vertex cover by Konig's theorem: 1 for its
 * vertices, as many as there are pairs); host memory, either may be NULL.  Not bipartite: mate all -1, cover all 0.
 * should_abort (may be NULL) is polled between phases; non-zero -> MGB200_ERR_ABORTED.  stats may be NULL. */
int mgb200_bipartite_matching_run(mgb200_bfs_graph *g, int (*should_abort)(void *user), void *abort_user,
                                  int64_t *mate_out, uint8_t *cover_out, mgb200_matching_stats *stats);
/* One shot on device 0: host COO (uint64 endpoints < n) -> the reference's answer. */
int mgb200_maximum_bipartite_matching(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                      uint64_t *matched_out);

/*
 * Strongly connected components on the same device graph: the partition of networkx.strongly_connected_components on
 * the MultiDiGraph of all vertices and edges (the reference's nxalg.strongly_connected_components).  Self-loops and
 * multi-edges change nothing.  component_out[v] is the number of v's component; components are numbered in the order
 * of their smallest vertex id, as in mgb200_wcc_run, so the output is canonical.  Multistep: a trim of the vertices
 * with no live in- or out-entry, a forward-backward search from a pivot, then colouring rounds; all integer work, so two
 * runs give byte-identical outputs and stats (run_ms aside).  A vertex's entries count in 32 bits (degree < 2^32).
 * Without a device every call fails with MGB200_ERR_CUDA.
 */
typedef struct mgb200_scc_stats {
  uint64_t components;        /* number of components                                                              */
  uint64_t largest_component; /* vertices in the largest one                                                       */
  uint64_t trimmed;           /* singleton components removed by the trim                                          */
  uint64_t pivot_component;   /* vertices of the component found by forward-backward from the pivot (0: none)      */
  uint64_t coloring_rounds;   /* colour-then-collect rounds after forward-backward                                 */
  uint64_t levels;            /* frontier levels of the forward, backward and propagation searches                 */
  uint64_t host_round_trips;  /* device-to-host waits of the run (trim levels, pivot, searches and colouring)       */
  uint64_t edges_inspected;   /* adjacency entries read: trim and searches together                                */
  double run_ms;              /* CUDA-event time, first kernel .. last label written (no transfers)                */
  uint64_t kernel_launches;
} mgb200_scc_stats;

/* component_out: n int64 values in host memory; stats may be NULL.  should_abort (may be NULL) is polled between host
 * round trips; non-zero -> MGB200_ERR_ABORTED and component_out is left untouched.  n == 0 returns MGB200_OK with zero
 * components and zero launches. */
int mgb200_scc_run(mgb200_bfs_graph *g, int (*should_abort)(void *user), void *abort_user, int64_t *component_out,
                   mgb200_scc_stats *stats);
/* One shot on device 0: host COO (uint64 endpoints < n) -> component_out[n] in host memory. */
int mgb200_strongly_connected_components(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                         int64_t *component_out);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* MGB200_BFS_H */

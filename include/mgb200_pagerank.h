/*
 * mgb200_pagerank.h -- C ABI of the GPU-native static-PageRank hot path.
 *
 * This is the boundary a host binds instead of the reference's CPU algorithm
 * (memgraph/memgraph @ 292f896a, all paths relative to the reference root):
 *
 *   reference interface                                              replaced by
 *   ---------------------------------------------------------------  ------------------------------------
 *   pagerank_alg::PageRankGraph(n, m, edges)                         mgb200_graph_create_host()
 *     mage/cpp/pagerank_module/algorithm/pagerank.hpp:40,            (COO in host memory -> device-resident
 *     pagerank.cpp:165-181                                            degree-sorted SELL-32 + segmented CSC)
 *   pagerank_alg::ParallelIterativePageRank(graph, max_iterations,   mgb200_pagerank_run()
 *     damping_factor, stop_epsilon, number_of_threads)               (power iteration as sm_90a kernels,
 *     pagerank.hpp:107-109, pagerank.cpp:193-240                      same recurrence / stop test / normalise)
 *   both, as called back to back by PagerankWrapper                  mgb200_parallel_iterative_pagerank()
 *     mage/cpp/pagerank_module/pagerank_module.cpp:100-102
 *
 * Plain pointers and sizes only; no C++ or torch types.  All functions return MGB200_OK (0) or an
 * MGB200_ERR_* code; mgb200_last_error() returns the calling thread's last message.  There is NO
 * CPU fallback: without a CUDA device every compute entry point fails with MGB200_ERR_CUDA.
 *
 * Thread-safety: distinct graph handles may be used from distinct threads concurrently (each
 * owns its stream and buffers); a single handle must not be used from two threads at once.
 */
#ifndef MGB200_PAGERANK_H
#define MGB200_PAGERANK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default) /* the library is built with -fvisibility=hidden */
#endif

#define MGB200_OK 0
#define MGB200_ERR_INVALID_ARGUMENT 1 /* bad pointer / endpoint >= n / unsupported size           */
#define MGB200_ERR_ZERO_THREADS 2     /* number_of_threads == 0 (reference: pagerank.cpp:63-65)     */
#define MGB200_ERR_CUDA 3             /* no device, out of device memory, launch or runtime failure */
#define MGB200_ERR_ABORTED 4          /* the should_abort callback asked to stop (mgp_must_abort)   */
#define MGB200_ERR_COMM 5             /* multi-GPU exchange set-up or peer time-out                 */

/* The reference's error text for number_of_threads == 0, kept verbatim for drop-in fidelity. */
#define MGB200_MSG_ZERO_THREADS "Number of threads can't be zero (0)!"

typedef struct mgb200_graph mgb200_graph; /* one device-resident partition of a graph */

typedef struct mgb200_graph_info {
  uint64_t node_count;     /* N, global                                               */
  uint64_t edge_count;     /* E, global (multi-edges and self-loops counted)          */
  uint32_t part_rank;      /* this partition's index                                  */
  uint32_t part_world;     /* number of partitions (GPUs)                             */
  uint64_t local_rows;     /* destination vertices owned by this partition            */
  uint64_t local_edges;    /* in-edges of the owned vertices                          */
  uint64_t heavy_rows;     /* rows with in-degree >= heavy threshold (segmented CSC)  */
  uint64_t heavy_edges;
  uint64_t heavy_segments;
  uint64_t sell_rows;      /* rows stored in SELL-32 slices                           */
  uint64_t sell_slices;
  uint64_t sell_entries;   /* 32 * sum(slice widths), padding included                */
  uint64_t zero_rows;      /* in-degree 0: rank is the constant (1-d)/N after iter 1  */
  uint64_t resident_bytes; /* device bytes held by the handle after build             */
  double build_ms;         /* device time of the CSR/SELL build                       */
  double upload_ms;        /* host COO -> device, wall clock (0 for create_device)    */
  uint64_t build_peak_bytes; /* device memory in use at the build's high-water mark   */
  uint64_t tiled_edges;    /* heavy-row edges gathered from shared-memory tiles       */
  uint64_t tile_chunks;    /* their (row, tile) runs of <= MGB200_TILE_CHUNK edges    */
  uint64_t block_edges;    /* in-edges from labels >= MGB200_BLOCK_FROM (block class) */
  uint64_t block_chunks;   /* their (row, label block) runs, <= MGB200_BLOCK_CHUNK    */
  uint64_t blocks;         /* label blocks with at least one chunk (one launch each)  */
  uint64_t tile_slices;    /* SELL-32 slices of tile chunks, tile-major               */
  uint64_t tile_runs;      /* contiguous slice runs the tile kernel's CTAs draw (MGB200_TILE_RUNS) */
  uint64_t table_labels;   /* hottest labels the SELL walk reads from shared memory (0: no table) */
  uint64_t stage_entries;  /* SELL entries read from values the block passes stage (MGB200_SELL_STAGE) */
} mgb200_graph_info;

typedef struct mgb200_run_stats {
  uint64_t iterations;  /* number_of_iterations of the reference loop (pagerank.cpp:230) */
  double last_diff;     /* max_v |r_k[v] - r_{k-1}[v]| of the last iteration (this partition set) */
  double rank_sum;      /* sum of un-normalised ranks (the NormalizeRank divisor)        */
  double iterate_ms;    /* CUDA-event time: first iteration kernel .. normalise done     */
  double kernel_ms;     /* CUDA-event time summed over the timed launches of the dominant (SELL)
                           kernel; 0 unless params.time_spmv_kernel                       */
  uint64_t kernel_timed_launches; /* how many launches kernel_ms covers (first <= 64)    */
  double class_ms[6];   /* per kernel class, summed over the timed iterations: 0 zero-rows, 1 SELL rows,
                           2 SELL epilogue (+peer push), 3 heavy segments, 4 heavy finish, 5 iteration end
                           (barrier + convergence test); classes may overlap in time                 */
  uint64_t kernel_launches; /* kernels launched inside the timed region                 */
  uint64_t spmv_launches;   /* launches of the dominant (SELL) kernel                    */
} mgb200_run_stats;

/* Optional cooperative-abort hook, polled between iteration batches (mg_procedure.h:1945-1962). */
typedef int (*mgb200_abort_fn)(void *user);

typedef struct mgb200_run_params {
  uint64_t max_iterations; /* size_t in the reference; negative int64 wraps (pagerank_module.cpp:95) */
  double damping_factor;
  double stop_epsilon;
  mgb200_abort_fn should_abort; /* may be NULL */
  void *abort_user;
  int rank_out_on_device;  /* 0: rank_out is host memory, 1: device memory on the graph's device */
  int time_spmv_kernel;    /* 1: bracket the dominant (SELL) kernel's launches with CUDA events on the
                              launching stream and report their summed duration in stats.kernel_ms  */
} mgb200_run_params;

const char *mgb200_last_error(void);
int mgb200_device_count(int *count_out);

/* ---- graph ingest (the PageRankGraph constructor's job) ---------------------------------------- */

/* COO in host memory, uint64 endpoints as in pagerank_alg::EdgePair (pagerank.hpp:24).  Endpoints
 * must be < n; n must be < 2^32 - 1.  part_rank/part_world select the vertex partition this handle
 * holds (0/1 for a single GPU). */
int mgb200_graph_create_host(int device, uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                             uint32_t part_rank, uint32_t part_world, mgb200_graph **out);

/* Same for callers that hold 32-bit dense ids already (the query module narrows while it pulls the graph through
 * the mgp iterators): half the host memory, nothing to narrow.  Both host forms stage through pinned, double-buffered
 * chunks filled by a few host threads (MGB200_INGEST_THREADS, default min(32, cores/2)) while the previous chunk is
 * on the wire: one pass, 8 bytes per edge over PCIe. */
int mgb200_graph_create_host_u32(int device, uint64_t n, uint64_t m, const uint32_t *from, const uint32_t *to,
                                 uint32_t part_rank, uint32_t part_world, mgb200_graph **out);

/* Host-only: 128-bit order-sensitive fingerprint of a dense COO.  The mgp ABI has no graph version, so a module that
 * wants to keep the device graph across CALLs (MGB200_GRAPH_CACHE=1 in pagerank.so) compares fingerprints of what it
 * pulled.  The value depends on MGB200_INGEST_THREADS (the partial hashes are combined per thread). */
int mgb200_coo_fingerprint_u32(uint64_t n, uint64_t m, const uint32_t *from, const uint32_t *to, uint64_t out[2]);

/* Same, COO already resident on `device` as uint32 (the inputs are read, not consumed). */
int mgb200_graph_create_device(int device, uint64_t n, uint64_t m, const uint32_t *d_from, const uint32_t *d_to,
                               uint32_t part_rank, uint32_t part_world, mgb200_graph **out);

void mgb200_graph_destroy(mgb200_graph *g);
int mgb200_graph_get_info(const mgb200_graph *g, mgb200_graph_info *info);

/* ---- the hot path (ParallelIterativePageRank) --------------------------------------------------- */

/* Single-partition run.  rank_out receives node_count doubles in ORIGINAL vertex-id order,
 * normalised to sum 1 (pagerank.cpp:156-161, :238). */
int mgb200_pagerank_run(mgb200_graph *g, const mgb200_run_params *params, double *rank_out,
                        mgb200_run_stats *stats);

/* One gather alone: y[v] = sum over the edges u -> v of x[u] (times the edge's weight when `weighted`), with the
 * kernels, layout and summation order every PageRank-layout algorithm iterates, and no epilogue.  x and y hold
 * node_count doubles in ORIGINAL vertex-id order, in host memory (on_device = 0) or on the graph's device (1).
 * Single-partition handles only; weighted = 1 needs a handle built with edge weights
 * (mgb200_graph_create_host_weighted_u32).  The call overwrites the handle's contribution buffer: a later run, Katz or
 * cuGraph-PageRank call on the handle starts from scratch, as it does anyway. */
int mgb200_graph_gather(mgb200_graph *g, const double *x, double *y, int on_device, int weighted);

/* PageRankGraph(n, m, edges) + ParallelIterativePageRank(graph, ...) in one call, host buffers in
 * and out -- what PagerankWrapper does between ingest and record emission
 * (pagerank_module.cpp:100-102).  number_of_threads is accepted for signature fidelity: 0 is the
 * reference's error, any other value is ignored (it only changes the reference's summation order). */
int mgb200_parallel_iterative_pagerank(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                       uint64_t max_iterations, double damping_factor, double stop_epsilon,
                                       uint32_t number_of_threads, double *rank_out, uint64_t *iterations_out);

/* Same call spread over `gpu_count` GPUs of this machine (devices[q], or ordinals 0..gpu_count-1 when
 * NULL): one partition and one host thread per GPU inside the call, peers wired by peer access. */
int mgb200_parallel_iterative_pagerank_multi(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                                             uint64_t max_iterations, double damping_factor, double stop_epsilon,
                                             uint32_t number_of_threads, uint32_t gpu_count, const int *devices,
                                             double *rank_out, uint64_t *iterations_out);

/* The same with a parameter block, so that the cooperative-abort hook works across GPUs too: should_abort is polled
 * from the CALLING thread only (Memgraph's mgp_must_abort must not be called from other threads, mg_procedure.h:75-81)
 * and the first request becomes a collective stop on all partitions -> MGB200_ERR_ABORTED.  rank_out is host memory. */
int mgb200_pagerank_multi(uint64_t n, uint64_t m, const uint64_t *from, const uint64_t *to,
                          const mgb200_run_params *params, uint32_t number_of_threads, uint32_t gpu_count,
                          const int *devices, double *rank_out, uint64_t *iterations_out);

int mgb200_pagerank_multi_u32(uint64_t n, uint64_t m, const uint32_t *from, const uint32_t *to,
                              const mgb200_run_params *params, uint32_t number_of_threads, uint32_t gpu_count,
                              const int *devices, double *rank_out, uint64_t *iterations_out);

/* ---- multi-GPU: one partition per GPU, contributions pushed to peers over NVLink --------------- */

#define MGB200_IPC_HANDLE_BYTES 64

/* Which global labels partition `part_rank` of `part_world` owns for an n-vertex graph: vertices sorted by degree are
 * dealt round-robin, each owner's share becomes one contiguous label range [first_label, first_label + rows).  Host-only
 * arithmetic (no device needed). */
int mgb200_partition_range(uint64_t n, uint32_t part_world, uint32_t part_rank, uint64_t *first_label_out,
                           uint64_t *rows_out);

/* The label <-> (owner, local row) arithmetic of both labellings, host-only (diagnostics and tests; the device code
 * uses the same functions, csrc/core.hpp RowMap).  global_order = 0: the dealt contiguous ranges above (heavy_rows is
 * ignored); 1: label = position in the global degree order, the first `heavy_rows` labels owned round-robin, then
 * blocks of 32 labels owned round-robin (MGB200_LABELLING=global).
 *   mgb200_partition_locate: label -> owning partition and its local row there;
 *   mgb200_partition_label : (part_rank, local_row) -> label; rows_out = number of local rows of part_rank. */
int mgb200_partition_locate(uint64_t n, uint64_t heavy_rows, uint32_t part_world, int global_order, uint64_t label,
                            uint32_t *owner_out, uint64_t *local_row_out);
int mgb200_partition_label(uint64_t n, uint64_t heavy_rows, uint32_t part_world, int global_order, uint32_t part_rank,
                           uint64_t local_row, uint64_t *label_out, uint64_t *rows_out);

/* Exports this partition's exchange window (contribution buffers + flag page) as a CUDA IPC
 * handle, for a peer PROCESS to open. */
int mgb200_graph_export_window(mgb200_graph *g, void *ipc_handle_out /* MGB200_IPC_HANDLE_BYTES */);
/* Connects the partition to its peers.  Exactly one of the two arrays is used per peer p != part_rank:
 * ipc_handles[p] (64-byte handle from another process) or, for peers in the SAME process,
 * peer_graphs[p].  Both arrays have part_world entries; unused entries are NULL. */
int mgb200_graph_connect_peers(mgb200_graph *g, const void *const *ipc_handles, mgb200_graph *const *peer_graphs);

/* Multi-partition run: every partition calls this (one process per GPU, or one host thread per
 * GPU).  The iteration loop, the max-diff / rank-sum reductions and the contribution exchange run
 * entirely on the devices over peer memory.  rank_out receives THIS partition's local_rows
 * normalised ranks; vertex_out (may be NULL) the original vertex id of each. */
int mgb200_pagerank_run_partition(mgb200_graph *g, const mgb200_run_params *params, double *rank_out,
                                  uint32_t *vertex_out, mgb200_run_stats *stats);

/* ---- synthetic workload (BASELINE.json configs; SURVEY 8d) -------------------------------------- */

/* RMAT(a, b, c, d = 1-a-b-c) edge list, edges [first_edge, first_edge + count) of a graph with
 * 2^scale vertices, counter-based (splitmix64 of seed, edge index, level pair) so the host and the
 * device produce identical bytes.  No clip-and-flip, no dedup, no id permutation. */
int mgb200_rmat_generate_device(int device, uint32_t scale, uint64_t first_edge, uint64_t count, uint64_t seed,
                                double a, double b, double c, uint32_t *d_from, uint32_t *d_to);
int mgb200_rmat_generate_host(uint32_t scale, uint64_t first_edge, uint64_t count, uint64_t seed, double a, double b,
                              double c, uint64_t *from, uint64_t *to);

/* A partition of the RMAT graph built straight from the generator, a chunk (2^27 edges) at a time, in two passes
 * (degrees, then the edges this partition owns): no device ever holds the whole edge list, so the graph a machine can
 * take grows with its GPU count -- every partition still SCANS all edges, it does not keep them. */
int mgb200_graph_create_rmat(int device, uint32_t scale, uint64_t edge_count, uint64_t seed, double a, double b, double c,
                             uint32_t part_rank, uint32_t part_world, mgb200_graph **out);

/* ---- small device-memory helpers so a ctypes caller needs nothing but this library -------------- */
int mgb200_device_malloc(int device, size_t bytes, void **ptr_out);
int mgb200_device_free(int device, void *ptr);
int mgb200_copy_to_device(int device, void *dst_device, const void *src_host, size_t bytes);
int mgb200_copy_to_host(int device, void *dst_host, const void *src_device, size_t bytes);
int mgb200_device_info(int device, char *name_out, size_t name_cap, int *sm_count, size_t *total_bytes);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* MGB200_PAGERANK_H */

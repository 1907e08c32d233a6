"""ctypes binding of include/mgb200_pagerank.h.  Fails loudly when the library is missing: the
product has no fallback (build with `python -m memgraph_b200.build` or __graft_entry__.build())."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MGB200_LIBRARY") or os.path.join(_HERE, "_build", "libmgb200_pagerank.so")

u64, u32, f64, i32 = ctypes.c_uint64, ctypes.c_uint32, ctypes.c_double, ctypes.c_int
vp = ctypes.c_void_p

OK, ERR_INVALID_ARGUMENT, ERR_ZERO_THREADS, ERR_CUDA, ERR_ABORTED, ERR_COMM = 0, 1, 2, 3, 4, 5
IPC_HANDLE_BYTES = 64


class GraphInfo(ctypes.Structure):
    _fields_ = [("node_count", u64), ("edge_count", u64), ("part_rank", u32), ("part_world", u32),
                ("local_rows", u64), ("local_edges", u64), ("heavy_rows", u64), ("heavy_edges", u64),
                ("heavy_segments", u64), ("sell_rows", u64), ("sell_slices", u64), ("sell_entries", u64),
                ("zero_rows", u64), ("resident_bytes", u64), ("build_ms", f64), ("upload_ms", f64), ("build_peak_bytes", u64),
                ("tiled_edges", u64), ("tile_chunks", u64),
                ("block_edges", u64), ("block_chunks", u64), ("blocks", u64),
                ("tile_slices", u64), ("tile_runs", u64), ("table_labels", u64),
                ("stage_entries", u64)]


class RunStatsC(ctypes.Structure):
    _fields_ = [("iterations", u64), ("last_diff", f64), ("rank_sum", f64), ("iterate_ms", f64), ("kernel_ms", f64),
                ("kernel_timed_launches", u64), ("class_ms", f64 * 6), ("kernel_launches", u64), ("spmv_launches", u64)]


class BfsStats(ctypes.Structure):
    _fields_ = [("levels", u32), ("top_down_levels", u32), ("bottom_up_levels", u32), ("reached", u64),
                ("edges_inspected", u64), ("traverse_ms", f64), ("kernel_launches", u64)]


class BcStats(ctypes.Structure):
    _fields_ = [("sources", u64), ("batches", u64), ("batch_width", u32), ("max_levels", u32), ("edges_traversed", u64),
                ("run_ms", f64), ("kernel_launches", u64)]


class WccStats(ctypes.Structure):
    _fields_ = [("components", u64), ("largest_component", u64), ("skipped_vertices", u64), ("edges_inspected", u64),
                ("run_ms", f64), ("kernel_launches", u64)]


class BiconnectivityStats(ctypes.Structure):
    _fields_ = [("trees", u64), ("forest_depth", u32), ("bridges", u64), ("components", u64), ("edges_inspected", u64),
                ("run_ms", f64), ("kernel_launches", u64)]


class WspStats(ctypes.Structure):
    _fields_ = [("rounds", u64), ("buckets", u64), ("hop_levels", u32), ("delta", f64), ("reached", u64),
                ("relaxations", u64), ("entries_inspected", u64), ("invalid_edge", u64), ("run_ms", f64),
                ("kernel_launches", u64)]


class MatchingStats(ctypes.Structure):
    _fields_ = [("bipartite", i32), ("left_vertices", u64), ("matched", u64), ("initial_matched", u64), ("phases", u64),
                ("max_levels", u32), ("edges_inspected", u64), ("run_ms", f64), ("kernel_launches", u64)]


class SccStats(ctypes.Structure):
    _fields_ = [("components", u64), ("largest_component", u64), ("trimmed", u64), ("pivot_component", u64),
                ("coloring_rounds", u64), ("levels", u64), ("host_round_trips", u64), ("edges_inspected", u64),
                ("run_ms", f64), ("kernel_launches", u64)]


class KatzStats(ctypes.Structure):
    _fields_ = [("iterations", u64), ("max_out_degree", u64), ("gamma", f64), ("iterate_ms", f64),
                ("kernel_launches", u64), ("tie_order_runs", u64)]


class CugraphParams(ctypes.Structure):
    _fields_ = [("max_iterations", u64), ("damping_factor", f64), ("stop_epsilon", f64), ("n_personalization", u64),
                ("personalization_vertices", vp), ("personalization_values", vp)]


class CugraphStats(ctypes.Structure):
    _fields_ = [("iterations", u64), ("converged", i32), ("last_diff_sum", f64), ("iterate_ms", f64),
                ("kernel_launches", u64)]


class HitsParams(ctypes.Structure):
    _fields_ = [("max_iterations", u64), ("tolerance", f64), ("normalized", i32)]


class HitsStats(ctypes.Structure):
    _fields_ = [("iterations", u64), ("converged", i32), ("last_diff_sum", f64), ("iterate_ms", f64),
                ("kernel_launches", u64)]


KATZ_NOT_CONVERGED = 16
ERR_INVALID_WEIGHT = 17
ABORT_FN = ctypes.CFUNCTYPE(ctypes.c_int, vp)


class RunParams(ctypes.Structure):
    _fields_ = [("max_iterations", u64), ("damping_factor", f64), ("stop_epsilon", f64), ("should_abort", ABORT_FN),
                ("abort_user", vp), ("rank_out_on_device", i32), ("time_spmv_kernel", i32)]


EXPORTS = {
    # name: (restype, argtypes) -- one entry per function declared in include/mgb200_pagerank.h
    "mgb200_last_error": (ctypes.c_char_p, []),
    "mgb200_device_count": (i32, [ctypes.POINTER(i32)]),
    "mgb200_graph_create_host": (i32, [i32, u64, u64, vp, vp, u32, u32, ctypes.POINTER(vp)]),
    "mgb200_graph_create_host_u32": (i32, [i32, u64, u64, vp, vp, u32, u32, ctypes.POINTER(vp)]),
    "mgb200_coo_fingerprint_u32": (i32, [u64, u64, vp, vp, vp]),
    "mgb200_graph_create_device": (i32, [i32, u64, u64, vp, vp, u32, u32, ctypes.POINTER(vp)]),
    "mgb200_graph_destroy": (None, [vp]),
    "mgb200_graph_get_info": (i32, [vp, ctypes.POINTER(GraphInfo)]),
    "mgb200_pagerank_run": (i32, [vp, ctypes.POINTER(RunParams), vp, ctypes.POINTER(RunStatsC)]),
    "mgb200_graph_gather": (i32, [vp, vp, vp, i32, i32]),
    "mgb200_parallel_iterative_pagerank": (i32, [u64, u64, vp, vp, u64, f64, f64, u32, vp, ctypes.POINTER(u64)]),
    "mgb200_parallel_iterative_pagerank_multi": (i32, [u64, u64, vp, vp, u64, f64, f64, u32, u32, vp, vp,
                                                       ctypes.POINTER(u64)]),
    "mgb200_pagerank_multi": (i32, [u64, u64, vp, vp, ctypes.POINTER(RunParams), u32, u32, vp, vp, ctypes.POINTER(u64)]),
    "mgb200_pagerank_multi_u32": (i32, [u64, u64, vp, vp, ctypes.POINTER(RunParams), u32, u32, vp, vp, ctypes.POINTER(u64)]),
    "mgb200_partition_range": (i32, [u64, u32, u32, ctypes.POINTER(u64), ctypes.POINTER(u64)]),
    "mgb200_partition_locate": (i32, [u64, u64, u32, i32, u64, ctypes.POINTER(u32), ctypes.POINTER(u64)]),
    "mgb200_partition_label": (i32, [u64, u64, u32, i32, u32, u64, ctypes.POINTER(u64), ctypes.POINTER(u64)]),
    "mgb200_graph_export_window": (i32, [vp, vp]),
    "mgb200_graph_connect_peers": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(vp)]),
    "mgb200_pagerank_run_partition": (i32, [vp, ctypes.POINTER(RunParams), vp, vp, ctypes.POINTER(RunStatsC)]),
    # include/mgb200_bfs.h
    "mgb200_bfs_graph_create_device": (i32, [i32, u64, u64, vp, vp, ctypes.POINTER(vp)]),
    "mgb200_bfs_graph_create_host": (i32, [i32, u64, u64, vp, vp, ctypes.POINTER(vp)]),
    "mgb200_bfs_graph_destroy": (None, [vp]),
    "mgb200_bfs_run": (i32, [vp, u64, i32, ctypes.c_int64, ctypes.c_int64, vp, i32, ctypes.POINTER(BfsStats)]),
    "mgb200_bc_run": (i32, [vp, i32, u64, u64, ABORT_FN, vp, vp, i32, ctypes.POINTER(BcStats)]),
    "mgb200_betweenness_centrality": (i32, [u64, u64, vp, vp, i32, i32, vp]),
    "mgb200_wcc_run": (i32, [vp, vp, ctypes.POINTER(WccStats)]),
    "mgb200_weakly_connected_components": (i32, [u64, u64, vp, vp, vp]),
    "mgb200_biconnectivity_run": (i32, [vp, u64, vp, vp, vp, vp, ctypes.POINTER(BiconnectivityStats)]),
    "mgb200_bridges": (i32, [u64, u64, vp, vp, vp]),
    "mgb200_biconnected_components": (i32, [u64, u64, vp, vp, vp]),
    "mgb200_bfs_graph_set_weights": (i32, [vp, u64, vp, vp, vp]),
    "mgb200_wsp_run": (i32, [vp, u64, i32, ctypes.c_int64, ABORT_FN, vp, vp, vp, ctypes.POINTER(WspStats)]),
    "mgb200_weighted_shortest_paths": (i32, [u64, u64, vp, vp, vp, u64, i32, ctypes.c_int64, vp, vp]),
    "mgb200_bipartite_matching_run": (i32, [vp, ABORT_FN, vp, vp, vp, ctypes.POINTER(MatchingStats)]),
    "mgb200_maximum_bipartite_matching": (i32, [u64, u64, vp, vp, ctypes.POINTER(u64)]),
    "mgb200_scc_run": (i32, [vp, ABORT_FN, vp, vp, ctypes.POINTER(SccStats)]),
    "mgb200_strongly_connected_components": (i32, [u64, u64, vp, vp, vp]),
    # include/mgb200_katz.h
    "mgb200_katz_run": (i32, [vp, f64, f64, u64, vp, ctypes.POINTER(KatzStats)]),
    "mgb200_katz_centrality": (i32, [u64, u64, vp, vp, f64, f64, u64, vp, ctypes.POINTER(u64)]),
    "mgb200_katz_tie_order": (i32, [u64, vp, vp]),
    # include/mgb200_personalized.h
    "mgb200_graph_create_host_weighted_u32": (i32, [i32, u64, u64, vp, vp, vp, ctypes.POINTER(vp)]),
    "mgb200_cugraph_pagerank_run": (i32, [vp, ctypes.POINTER(CugraphParams), vp, ctypes.POINTER(CugraphStats)]),
    "mgb200_hits_graph_create_host_u32": (i32, [i32, u64, u64, vp, vp, ctypes.POINTER(vp)]),
    "mgb200_hits_graph_get_info": (i32, [vp, ctypes.POINTER(GraphInfo), ctypes.POINTER(GraphInfo)]),
    "mgb200_hits_graph_destroy": (None, [vp]),
    "mgb200_hits_run": (i32, [vp, ctypes.POINTER(HitsParams), vp, vp, ctypes.POINTER(HitsStats)]),
    "mgb200_hits": (i32, [u64, u64, vp, vp, ctypes.POINTER(HitsParams), vp, vp, ctypes.POINTER(HitsStats)]),
    "mgb200_graph_create_rmat": (i32, [i32, u32, u64, u64, f64, f64, f64, u32, u32, ctypes.POINTER(vp)]),
    "mgb200_rmat_generate_device": (i32, [i32, u32, u64, u64, u64, f64, f64, f64, vp, vp]),
    "mgb200_rmat_generate_host": (i32, [u32, u64, u64, u64, f64, f64, f64, vp, vp]),
    "mgb200_device_malloc": (i32, [i32, ctypes.c_size_t, ctypes.POINTER(vp)]),
    "mgb200_device_free": (i32, [i32, vp]),
    "mgb200_copy_to_device": (i32, [i32, vp, vp, ctypes.c_size_t]),
    "mgb200_copy_to_host": (i32, [i32, vp, vp, ctypes.c_size_t]),
    "mgb200_device_info": (i32, [i32, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(i32),
                                 ctypes.POINTER(ctypes.c_size_t)]),
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: the CUDA extension is required (no CPU fallback). "
                "Build it with `python -m memgraph_b200.build`.")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in EXPORTS.items():
            fn = getattr(L, name)  # AttributeError if the library does not export what the header declares
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib

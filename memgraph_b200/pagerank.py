"""Host-side mirror of the reference's PageRank interface over the C ABI (see package docstring)."""
import ctypes
from dataclasses import dataclass

import numpy as np

from . import _native as N


class MgB200Error(RuntimeError):
    def __init__(self, code, message):
        super().__init__(message)
        self.code = code


def _check(rc):
    if rc != N.OK:
        raise MgB200Error(rc, N.lib().mgb200_last_error().decode(errors="replace"))


def device_count():
    n = ctypes.c_int(0)
    _check(N.lib().mgb200_device_count(ctypes.byref(n)))
    return n.value


@dataclass
class RunStats:
    iterations: int
    last_diff: float
    rank_sum: float
    iterate_ms: float
    kernel_ms: float
    kernel_timed_launches: int
    class_ms: tuple
    kernel_launches: int
    spmv_launches: int


def _stats(c):
    return RunStats(c.iterations, c.last_diff, c.rank_sum, c.iterate_ms, c.kernel_ms, c.kernel_timed_launches,
                    tuple(c.class_ms), c.kernel_launches, c.spmv_launches)


def make_params(max_iterations, damping_factor, stop_epsilon, on_device=False, time_spmv_kernel=False,
                should_abort=None):
    p = N.RunParams()
    p.max_iterations = int(max_iterations) & (2**64 - 1)  # int64 -> size_t wrap, pagerank_module.cpp:95
    p.damping_factor = float(damping_factor)
    p.stop_epsilon = float(stop_epsilon)
    cb = N.ABORT_FN(lambda _u: 1 if should_abort() else 0) if should_abort else N.ABORT_FN()
    p.should_abort = cb
    p.rank_out_on_device = 1 if on_device else 0
    p.time_spmv_kernel = 1 if time_spmv_kernel else 0
    return p, cb  # keep cb alive for the duration of the call


class PageRankGraph:
    """Device-resident counterpart of pagerank_alg::PageRankGraph (pagerank.hpp:31-76).

    ``PageRankGraph(number_of_nodes, number_of_edges, edges)`` takes the reference constructor's
    arguments (pagerank.hpp:40): ``edges`` is a sequence / (m, 2) array of (source, target) pairs with
    ids in [0, number_of_nodes); self-loops and multi-edges count.  ``number_of_edges`` must equal
    ``len(edges)`` (the reference reads past the vector otherwise, pagerank.cpp:68,91).
    Alternative constructors: :meth:`from_arrays` (two host arrays) and :meth:`from_device`
    (uint32 COO already on the GPU, e.g. from :func:`rmat_edges_device`).
    """

    def __init__(self, number_of_nodes, number_of_edges, edges, device=0, part_rank=0, part_world=1):
        e = np.asarray(edges, dtype=np.uint64).reshape(-1, 2)
        if int(number_of_edges) != len(e):
            raise MgB200Error(N.ERR_INVALID_ARGUMENT, "number_of_edges must equal len(edges)")
        self._init_host(int(number_of_nodes), np.ascontiguousarray(e[:, 0]), np.ascontiguousarray(e[:, 1]), device,
                        part_rank, part_world)

    @classmethod
    def from_arrays(cls, number_of_nodes, sources, targets, device=0, part_rank=0, part_world=1):
        self = cls.__new__(cls)
        s = np.ascontiguousarray(sources, dtype=np.uint64)
        t = np.ascontiguousarray(targets, dtype=np.uint64)
        if s.shape != t.shape or s.ndim != 1:
            raise MgB200Error(N.ERR_INVALID_ARGUMENT, "sources and targets must be 1-D arrays of equal length")
        self._init_host(int(number_of_nodes), s, t, device, part_rank, part_world)
        return self

    @classmethod
    def from_device(cls, number_of_nodes, number_of_edges, d_sources_ptr, d_targets_ptr, device=0, part_rank=0,
                    part_world=1):
        """uint32 COO resident on ``device`` (raw device pointers, e.g. tensor.data_ptr())."""
        self = cls.__new__(cls)
        h = N.vp()
        _check(N.lib().mgb200_graph_create_device(device, int(number_of_nodes), int(number_of_edges),
                                                  d_sources_ptr, d_targets_ptr, part_rank, part_world,
                                                  ctypes.byref(h)))
        self._finish(h, device)
        return self

    def _init_host(self, n, s, t, device, part_rank, part_world):
        h = N.vp()
        _check(N.lib().mgb200_graph_create_host(device, n, len(s), s.ctypes.data, t.ctypes.data, part_rank, part_world,
                                                ctypes.byref(h)))
        self._finish(h, device)

    @classmethod
    def from_rmat(cls, scale, number_of_edges=None, seed=42, device=0, part_rank=0, part_world=1, a=0.57, b=0.19, c=0.19):
        """The synthetic RMAT graph (SURVEY 8d) built straight from the generator, a chunk at a time: no device holds the
        whole edge list (mgb200_graph_create_rmat)."""
        self = cls.__new__(cls)
        h = N.vp()
        m = (16 << scale) if number_of_edges is None else int(number_of_edges)
        _check(N.lib().mgb200_graph_create_rmat(device, int(scale), m, int(seed), a, b, c, part_rank, part_world,
                                                ctypes.byref(h)))
        self._finish(h, device)
        return self

    def _finish(self, h, device):
        self._h = h
        self.device = device
        info = N.GraphInfo()
        _check(N.lib().mgb200_graph_get_info(h, ctypes.byref(info)))
        self.info = {k: getattr(info, k) for k, _ in N.GraphInfo._fields_}

    # names follow pagerank.hpp:47-59
    def get_node_count(self):
        return self.info["node_count"]

    def get_edge_count(self):
        return self.info["edge_count"]

    @property
    def handle(self):
        return self._h

    def close(self):
        if getattr(self, "_h", None):
            N.lib().mgb200_graph_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def run(self, max_iterations=100, damping_factor=0.85, stop_epsilon=1e-5, out_device_ptr=None,
            time_spmv_kernel=False, should_abort=None, out=None):
        """The iteration proper (pagerank.cpp:193-240) on this graph.  Returns (ranks, RunStats); ranks is
        a host float64 array in original vertex order (``out`` if given, e.g. a pinned buffer), or None
        when ``out_device_ptr`` receives them on the device."""
        p, _cb = make_params(max_iterations, damping_factor, stop_epsilon, out_device_ptr is not None,
                             time_spmv_kernel, should_abort)
        st = N.RunStatsC()
        n = self.get_node_count()
        if out_device_ptr is not None:
            _check(N.lib().mgb200_pagerank_run(self._h, ctypes.byref(p), out_device_ptr, ctypes.byref(st)))
            return None, _stats(st)
        if out is None:
            out = np.empty(n, dtype=np.float64)
        assert out.dtype == np.float64 and out.size >= n and out.flags["C_CONTIGUOUS"]
        _check(N.lib().mgb200_pagerank_run(self._h, ctypes.byref(p), out.ctypes.data if n else None,
                                           ctypes.byref(st)))
        return out, _stats(st)

    def gather(self, x, weighted=False):
        """y = A^T x through the gather every algorithm on this layout iterates (mgb200_graph_gather): ``y[v]`` is the
        sum of ``x[u]`` over the edges u -> v, each times its weight when ``weighted``.  ``x`` and the returned float64
        array are in original vertex order.  Single-partition handles only."""
        n = self.get_node_count()
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.shape != (n,):
            raise MgB200Error(N.ERR_INVALID_ARGUMENT, f"x must hold {n} values")
        y = np.empty(n, dtype=np.float64)
        _check(N.lib().mgb200_graph_gather(self._h, x.ctypes.data if n else None, y.ctypes.data if n else None, 0,
                                           1 if weighted else 0))
        return y

    # ---- multi-GPU: one partition per GPU (mgb200_pagerank.h "multi-GPU" section) ----------------------

    def export_window(self):
        """CUDA IPC handle (64 bytes) of this partition's exchange window, for a peer PROCESS."""
        buf = ctypes.create_string_buffer(N.IPC_HANDLE_BYTES)
        _check(N.lib().mgb200_graph_export_window(self._h, buf))
        return buf.raw

    def connect_peers(self, ipc_handles=None, local_graphs=None):
        """Wire this partition to its peers: ``ipc_handles[q]`` = bytes from peer process q, or
        ``local_graphs[q]`` = a PageRankGraph of the same process (entry for the own rank is ignored)."""
        world = self.info["part_world"]
        harr = (N.vp * world)()
        garr = (N.vp * world)()
        keep = []
        for q in range(world):
            if q == self.info["part_rank"]:
                continue
            if local_graphs is not None and local_graphs[q] is not None:
                garr[q] = local_graphs[q].handle
            elif ipc_handles is not None and ipc_handles[q] is not None:
                b = ctypes.create_string_buffer(bytes(ipc_handles[q]), N.IPC_HANDLE_BYTES)
                keep.append(b)
                harr[q] = ctypes.cast(b, N.vp)
        _check(N.lib().mgb200_graph_connect_peers(self._h, harr, garr))

    def run_partition(self, max_iterations=100, damping_factor=0.85, stop_epsilon=1e-5, time_spmv_kernel=False,
                      out_device_ptr=None, should_abort=None):
        """Every partition calls this concurrently.  Returns (ranks, vertices, RunStats) for the rows this
        partition owns: normalised ranks and the ORIGINAL vertex id of each (None, None when
        ``out_device_ptr`` receives the ranks on the device)."""
        p, _cb = make_params(max_iterations, damping_factor, stop_epsilon, out_device_ptr is not None,
                             time_spmv_kernel, should_abort)
        st = N.RunStatsC()
        rows = self.info["local_rows"]
        if out_device_ptr is not None:
            _check(N.lib().mgb200_pagerank_run_partition(self._h, ctypes.byref(p), out_device_ptr, None,
                                                         ctypes.byref(st)))
            return None, None, _stats(st)
        ranks = np.empty(rows, dtype=np.float64)
        verts = np.empty(rows, dtype=np.uint32)
        _check(N.lib().mgb200_pagerank_run_partition(self._h, ctypes.byref(p), ranks.ctypes.data if rows else None,
                                                     verts.ctypes.data if rows else None, ctypes.byref(st)))
        return ranks, verts, _stats(st)


def parallel_iterative_pagerank(graph, max_iterations=100, damping_factor=0.85, stop_epsilon=1e-5,
                                number_of_threads=1):
    """pagerank_alg::ParallelIterativePageRank (pagerank.hpp:107-109).  ``number_of_threads`` is kept
    for signature fidelity: 0 raises the reference's error, anything else is ignored on the GPU."""
    if (int(number_of_threads) & 0xFFFFFFFF) == 0:
        raise MgB200Error(N.ERR_ZERO_THREADS, "Number of threads can't be zero (0)!")
    ranks, _ = graph.run(max_iterations, damping_factor, stop_epsilon)
    return ranks


def pagerank_from_edges(n, sources, targets, max_iterations=100, damping_factor=0.85, stop_epsilon=1e-5,
                        number_of_threads=1, gpus=1):
    """One-call form (mgb200_parallel_iterative_pagerank[_multi]): host COO in, host ranks out."""
    s = np.ascontiguousarray(sources, dtype=np.uint64)
    t = np.ascontiguousarray(targets, dtype=np.uint64)
    out = np.empty(int(n), dtype=np.float64)
    it = ctypes.c_uint64(0)
    _check(N.lib().mgb200_parallel_iterative_pagerank_multi(
        int(n), len(s), s.ctypes.data, t.ctypes.data, int(max_iterations) & (2**64 - 1), float(damping_factor),
        float(stop_epsilon), int(number_of_threads) & 0xFFFFFFFF, int(gpus), None, out.ctypes.data if n else None,
        ctypes.byref(it)))
    return out, it.value


RMAT_A, RMAT_B, RMAT_C = 0.57, 0.19, 0.19  # graph_generator.cu:143-145


def rmat_edges_host(scale, count, seed=42, first_edge=0, a=RMAT_A, b=RMAT_B, c=RMAT_C):
    s = np.empty(count, dtype=np.uint64)
    t = np.empty(count, dtype=np.uint64)
    _check(N.lib().mgb200_rmat_generate_host(scale, first_edge, count, seed, a, b, c, s.ctypes.data, t.ctypes.data))
    return s, t


def rmat_edges_device(scale, count, d_sources_ptr, d_targets_ptr, seed=42, first_edge=0, device=0, a=RMAT_A, b=RMAT_B,
                      c=RMAT_C):
    _check(N.lib().mgb200_rmat_generate_device(device, scale, first_edge, count, seed, a, b, c, d_sources_ptr,
                                               d_targets_ptr))

"""Host-side mirror of the breadth-first expansion (include/mgb200_bfs.h): the arithmetic of
`MATCH (a)-[*BFS lower..upper]->(b)` (SingleSourceShortestPathCursor, src/query/plan/operator.cpp:2692-2912), and of
the weighted shortest path expansion `MATCH (a)-[*WSHORTEST ..u (e, n | e.w) total_weight]->(b)`
(ExpandWeightedShortestPathCursor, :2917-3267) on the same device graph."""
import ctypes

import numpy as np

from . import _native as N
from .pagerank import MgB200Error, _check

OUT, IN, BOTH = 0, 1, 2  # EdgeAtom::Direction
INT64_MAX = 2**63 - 1


class InvalidWeight(MgB200Error):
    """An edge weight the expansion evaluates is negative or not a number.  ``edge_index`` is the smallest COO index
    (in the order given to :meth:`BfsGraph.set_weights`) among the evaluated invalid edges; ``stats`` is the run's."""

    def __init__(self, message, edge_index, stats):
        super().__init__(N.ERR_INVALID_WEIGHT, message)
        self.edge_index, self.stats = edge_index, stats


class BfsGraph:
    """Device-resident CSR + CSC for traversals."""

    def __init__(self, number_of_nodes, sources, targets, device=0):
        s = np.ascontiguousarray(sources, dtype=np.uint64)
        t = np.ascontiguousarray(targets, dtype=np.uint64)
        h = N.vp()
        _check(N.lib().mgb200_bfs_graph_create_host(device, int(number_of_nodes), len(s), s.ctypes.data, t.ctypes.data,
                                                    ctypes.byref(h)))
        self._h, self.n, self.m = h, int(number_of_nodes), len(s)

    @classmethod
    def from_device(cls, number_of_nodes, number_of_edges, d_sources_ptr, d_targets_ptr, device=0):
        self = cls.__new__(cls)
        h = N.vp()
        _check(N.lib().mgb200_bfs_graph_create_device(device, int(number_of_nodes), int(number_of_edges), d_sources_ptr,
                                                      d_targets_ptr, ctypes.byref(h)))
        self._h, self.n, self.m = h, int(number_of_nodes), int(number_of_edges)
        return self

    def distances(self, source, direction=OUT, lower_bound=1, upper_bound=INT64_MAX):
        """depth at which the reference emits each vertex, -1 where it does not; returns (int32[n], stats dict)."""
        out = np.empty(self.n, dtype=np.int32)
        st = N.BfsStats()
        _check(N.lib().mgb200_bfs_run(self._h, int(source), int(direction), int(lower_bound), int(upper_bound),
                                      out.ctypes.data if self.n else None, 0, ctypes.byref(st)))
        return out, {k: getattr(st, k) for k, _ in N.BfsStats._fields_}

    def set_weights(self, sources, targets, weights):
        """One weight per edge of the COO the graph was built from (same pairs; NaN or negative = invalid)."""
        s = np.ascontiguousarray(sources, dtype=np.uint64)
        t = np.ascontiguousarray(targets, dtype=np.uint64)
        w = np.ascontiguousarray(weights, dtype=np.float64)
        if not (len(s) == len(t) == len(w)):
            raise MgB200Error(N.ERR_INVALID_ARGUMENT, "sources, targets and weights must have equal lengths")
        _check(N.lib().mgb200_bfs_graph_set_weights(self._h, len(s), s.ctypes.data if len(s) else None,
                                                    t.ctypes.data if len(s) else None,
                                                    w.ctypes.data if len(s) else None))

    def weighted_distances(self, source, direction=OUT, upper_bound=None, should_abort=None):
        """total_weight and hops of every vertex the weighted shortest path expansion produces (NaN / -1 elsewhere,
        the source included); upper_bound None = unbounded.  -> (float64[n], int32[n], stats dict).
        Raises InvalidWeight when an evaluated edge weight is negative or NaN."""
        dist = np.empty(self.n, dtype=np.float64)
        hops = np.empty(self.n, dtype=np.int32)
        st = N.WspStats()
        cb = N.ABORT_FN(lambda _user: 1 if should_abort() else 0) if should_abort else N.ABORT_FN()
        ub = INT64_MAX if upper_bound is None else int(upper_bound)
        rc = N.lib().mgb200_wsp_run(self._h, int(source), int(direction), ub, cb, None,
                                    dist.ctypes.data if self.n else None, hops.ctypes.data if self.n else None,
                                    ctypes.byref(st))
        stats = {k: getattr(st, k) for k, _ in N.WspStats._fields_}
        if rc == N.ERR_INVALID_WEIGHT:
            raise InvalidWeight(N.lib().mgb200_last_error().decode(errors="replace"), stats["invalid_edge"], stats)
        _check(rc)
        return dist, hops, stats

    def close(self):
        if getattr(self, "_h", None):
            N.lib().mgb200_bfs_graph_destroy(self._h)
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


def weighted_shortest_paths(n, sources, targets, weights, source, direction=OUT, upper_bound=None):
    """One shot on device 0 (mgb200_weighted_shortest_paths): -> (total_weight float64[n], hops int32[n])."""
    s = np.ascontiguousarray(sources, dtype=np.uint64)
    t = np.ascontiguousarray(targets, dtype=np.uint64)
    w = np.ascontiguousarray(weights, dtype=np.float64)
    dist, hops = np.empty(int(n), dtype=np.float64), np.empty(int(n), dtype=np.int32)
    rc = N.lib().mgb200_weighted_shortest_paths(int(n), len(s), s.ctypes.data, t.ctypes.data, w.ctypes.data,
                                                int(source), int(direction),
                                                INT64_MAX if upper_bound is None else int(upper_bound),
                                                dist.ctypes.data if n else None, hops.ctypes.data if n else None)
    if rc == N.ERR_INVALID_WEIGHT:
        raise InvalidWeight(N.lib().mgb200_last_error().decode(errors="replace"), None, None)
    _check(rc)
    return dist, hops


def splitmix_weights(m, kind="uniform"):
    """Seeded edge weights from splitmix64 of the edge index: "uniform" = [0, 1) with a 53-bit mantissa,
    "int" = integers 1..16 (as float64)."""
    with np.errstate(over="ignore"):
        z = (np.arange(1, int(m) + 1, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    if kind == "int":
        return (z % np.uint64(16) + np.uint64(1)).astype(np.float64)
    return (z >> np.uint64(11)).astype(np.float64) * 2.0**-53

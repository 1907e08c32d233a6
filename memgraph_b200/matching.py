"""Maximum bipartite matching on the device (include/mgb200_bfs.h): the host-side mirror of the reference's
``bipartite_matching.max`` (mage/cpp/bipartite_matching_module).  It runs on a :class:`memgraph_b200.bfs.BfsGraph`
handle -- the same device-resident CSR + CSC as BFS, betweenness and connectivity."""
import ctypes

import numpy as np

from . import _native as N
from .bfs import BfsGraph
from .pagerank import _check


def bipartite_matching_run(graph, should_abort=None):
    """A maximum matching of the undirected view and a minimum vertex cover of the same size (Konig's theorem):
    -> (int64[n] partner or -1, uint8[n] cover flags, stats dict).  Not bipartite (a self-loop or an odd cycle):
    stats["bipartite"] == 0, no pairs, an empty cover.  should_abort: optional callable polled between phases; when it
    returns True the call raises MgB200Error."""
    n = graph.n
    mate, cover = np.full(n, -1, dtype=np.int64), np.zeros(n, dtype=np.uint8)
    st = N.MatchingStats()
    cb = N.ABORT_FN(lambda _user: 1 if should_abort() else 0) if should_abort else N.ABORT_FN()
    _check(N.lib().mgb200_bipartite_matching_run(graph._h, cb, None, mate.ctypes.data if n else None,
                                                 cover.ctypes.data if n else None, ctypes.byref(st)))
    return mate, cover, {k: getattr(st, k) for k, _ in N.MatchingStats._fields_}


def maximum_bipartite_matching(n, sources, targets):
    """The reference procedure's answer end to end (device 0): the size of a maximum matching, 0 when the graph has a
    self-loop or an odd cycle."""
    s = np.ascontiguousarray(sources, dtype=np.uint64)
    t = np.ascontiguousarray(targets, dtype=np.uint64)
    out = ctypes.c_uint64(0)
    _check(N.lib().mgb200_maximum_bipartite_matching(int(n), len(s), s.ctypes.data, t.ctypes.data, ctypes.byref(out)))
    return int(out.value)


__all__ = ["BfsGraph", "bipartite_matching_run", "maximum_bipartite_matching"]

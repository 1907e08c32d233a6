"""Weakly connected components on the device (include/mgb200_bfs.h): the host-side mirror of the reference's
``weakly_connected_components.get`` (mage/cpp/connectivity_module/connectivity_module.cpp:41-84).  Runs on a
:class:`memgraph_b200.bfs.BfsGraph` handle -- the same device-resident CSR + CSC as BFS and betweenness."""
import ctypes

import numpy as np

from . import _native as N
from .bfs import BfsGraph
from .pagerank import _check


def wcc_run(graph):
    """Component number of every vertex, numbered in the order of each component's smallest vertex id.
    -> (int64[n], stats dict)."""
    out = np.zeros(graph.n, dtype=np.int64)
    st = N.WccStats()
    _check(N.lib().mgb200_wcc_run(graph._h, out.ctypes.data if graph.n else None, ctypes.byref(st)))
    return out, {k: getattr(st, k) for k, _ in N.WccStats._fields_}


def weakly_connected_components(n, sources, targets):
    """The reference procedure's numbering end to end (device 0): -> int64[n] in vertex-id order."""
    s = np.ascontiguousarray(sources, dtype=np.uint64)
    t = np.ascontiguousarray(targets, dtype=np.uint64)
    out = np.zeros(int(n), dtype=np.int64)
    _check(N.lib().mgb200_weakly_connected_components(int(n), len(s), s.ctypes.data, t.ctypes.data,
                                                      out.ctypes.data if n else None))
    return out


__all__ = ["BfsGraph", "wcc_run", "weakly_connected_components"]

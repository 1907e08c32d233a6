"""Connectivity on the device (include/mgb200_bfs.h): the host-side mirrors of the reference's
``weakly_connected_components.get`` (mage/cpp/connectivity_module/connectivity_module.cpp:41-84), ``bridges.get`` and
``biconnected_components.get`` (mage/cpp/bridges_module, mage/cpp/biconnected_components_module), and the strongly
connected components of ``nxalg.strongly_connected_components`` (query_modules/nxalg.py).  They run on a
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


def scc_run(graph, should_abort=None):
    """Strongly connected component of every vertex, numbered in the order of each component's smallest vertex id.
    ``should_abort`` (a callable returning true to stop) is polled between host round trips; a stop raises
    MgB200Error with code ERR_ABORTED.  -> (int64[n], stats dict)."""
    out = np.zeros(graph.n, dtype=np.int64)
    st = N.SccStats()
    cb = N.ABORT_FN(lambda _user: 1 if should_abort() else 0) if should_abort else N.ABORT_FN()
    _check(N.lib().mgb200_scc_run(graph._h, cb, None, out.ctypes.data if graph.n else None, ctypes.byref(st)))
    return out, {k: getattr(st, k) for k, _ in N.SccStats._fields_}


def strongly_connected_components(n, sources, targets):
    """One shot on device 0: int64[n] strongly connected component of every vertex, numbered in the order of each
    component's smallest vertex id."""
    s, t = _coo(sources, targets)
    out = np.zeros(int(n), dtype=np.int64)
    _check(N.lib().mgb200_strongly_connected_components(int(n), len(s), s.ctypes.data, t.ctypes.data,
                                                        out.ctypes.data if n else None))
    return out


def _coo(sources, targets):
    return np.ascontiguousarray(sources, dtype=np.uint64), np.ascontiguousarray(targets, dtype=np.uint64)


def biconnectivity_run(graph, sources, targets):
    """Bridge flags and biconnected components of every edge of the COO the graph was built from (same order):
    -> (uint8[m] bridge flags, int64[m] component numbers, -1 for self-loops, stats dict).  Components are numbered in
    the order of their first edge."""
    s, t = _coo(sources, targets)
    m = len(s)
    bridge, bcc = np.zeros(m, dtype=np.uint8), np.zeros(m, dtype=np.int64)
    st = N.BiconnectivityStats()
    _check(N.lib().mgb200_biconnectivity_run(graph._h, m, s.ctypes.data if m else None, t.ctypes.data if m else None,
                                             bridge.ctypes.data if m else None, bcc.ctypes.data if m else None,
                                             ctypes.byref(st)))
    return bridge, bcc, {k: getattr(st, k) for k, _ in N.BiconnectivityStats._fields_}


def bridges(n, sources, targets):
    """One shot on device 0: uint8[m], 1 where the edge is a bridge of the undirected multigraph."""
    s, t = _coo(sources, targets)
    out = np.zeros(len(s), dtype=np.uint8)
    _check(N.lib().mgb200_bridges(int(n), len(s), s.ctypes.data, t.ctypes.data, out.ctypes.data if len(s) else None))
    return out


def biconnected_components(n, sources, targets):
    """One shot on device 0: int64[m] biconnected component of every edge (-1 for self-loops), numbered in the order of
    each component's first edge."""
    s, t = _coo(sources, targets)
    out = np.zeros(len(s), dtype=np.int64)
    _check(N.lib().mgb200_biconnected_components(int(n), len(s), s.ctypes.data, t.ctypes.data,
                                                 out.ctypes.data if len(s) else None))
    return out


__all__ = ["BfsGraph", "wcc_run", "weakly_connected_components", "biconnectivity_run", "bridges",
           "biconnected_components", "scc_run", "strongly_connected_components"]

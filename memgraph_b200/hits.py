"""HITS hubs and authorities on the device (include/mgb200_personalized.h): the host-side mirror of what
``cugraph.hits.get`` computes (mage/cpp/cugraph_module/algorithms/hits.cu).  One :class:`HitsGraph` holds both
directions of a COO -- the forward layout gathers authorities, the reverse one hubs -- on one GPU."""
import ctypes

import numpy as np

from . import _native as N
from .pagerank import MgB200Error, _check


def _params(max_iterations, tolerance, normalized):
    p = N.HitsParams()
    p.max_iterations = int(max_iterations) & (2**64 - 1)  # INTEGER -> size_t wrap, as the reference module casts
    p.tolerance = float(tolerance)
    p.normalized = 1 if normalized else 0
    return p


def _stats(st):
    return {f: getattr(st, f) for f, _ in N.HitsStats._fields_}


def _coo(sources, targets):
    s = np.ascontiguousarray(sources, dtype=np.uint32)
    t = np.ascontiguousarray(targets, dtype=np.uint32)
    if s.shape != t.shape or s.ndim != 1:
        raise MgB200Error(N.ERR_INVALID_ARGUMENT, "sources and targets must be 1-D arrays of equal length")
    return s, t


class HitsGraph:
    """``HitsGraph(n, sources, targets, device=0)``: dense ids in [0, n); multi-edges and self-loops count.
    ``.info`` = (forward layout, reverse layout) as dicts of ``mgb200_graph_info``."""

    def __init__(self, n, sources, targets, device=0):
        s, t = _coo(sources, targets)
        h = N.vp()
        _check(N.lib().mgb200_hits_graph_create_host_u32(int(device), int(n), len(s), s.ctypes.data, t.ctypes.data,
                                                         ctypes.byref(h)))
        self._h = h
        self.n = int(n)
        self.device = device
        fwd, rev = N.GraphInfo(), N.GraphInfo()
        _check(N.lib().mgb200_hits_graph_get_info(h, ctypes.byref(fwd), ctypes.byref(rev)))
        self.info = tuple({k: getattr(i, k) for k, _ in N.GraphInfo._fields_} for i in (fwd, rev))

    def run(self, max_iterations=100, tolerance=1e-5, normalized=True):
        """-> (hubs[n], authorities[n] in original vertex order, stats dict)."""
        p = _params(max_iterations, tolerance, normalized)
        hubs = np.zeros(self.n, dtype=np.float64)
        auth = np.zeros(self.n, dtype=np.float64)
        st = N.HitsStats()
        _check(N.lib().mgb200_hits_run(self._h, ctypes.byref(p), hubs.ctypes.data if self.n else None,
                                       auth.ctypes.data if self.n else None, ctypes.byref(st)))
        return hubs, auth, _stats(st)

    def close(self):
        if getattr(self, "_h", None):
            N.lib().mgb200_hits_graph_destroy(self._h)
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


def hits(n, sources, targets, max_iterations=100, tolerance=1e-5, normalized=True):
    """One call (mgb200_hits, device MGB200_DEVICE or 0): -> (hubs, authorities, stats dict)."""
    s, t = _coo(sources, targets)
    p = _params(max_iterations, tolerance, normalized)
    hubs = np.zeros(int(n), dtype=np.float64)
    auth = np.zeros(int(n), dtype=np.float64)
    st = N.HitsStats()
    _check(N.lib().mgb200_hits(int(n), len(s), s.ctypes.data, t.ctypes.data, ctypes.byref(p),
                               hubs.ctypes.data if n else None, auth.ctypes.data if n else None, ctypes.byref(st)))
    return hubs, auth, _stats(st)

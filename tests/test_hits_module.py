"""cugraph.hits.so (memgraph_b200/csrc/cugraph_modules.cpp built with MGB200_CUGRAPH_HITS=1): the stand-in for the
reference's cuGraph HITS query module, on the BOOLEAN-capable in-memory mgp host plus a call that returns two named
FLOAT columns (tests/mgp_hits_host.cpp).  That host defines the same mgp_* symbols as the other hosts, so the tests
that load it run in a child interpreter (@isolated, tests/_bc_host.py).  No-GPU part: exports and imports, the
registered signature, argument typing, graphs that need no device, loud failure without a device.  GPU part (-m gpu):
the reference's e2e fixtures through the module, rows in ascending gid, vanished vertices in both modes."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import conftest
from _bc_host import REPO, isolated
from test_hits_oracle import FIXTURES, check_fixture, oracle_hits

HITS_MODULE_SO = os.path.join(REPO, "memgraph_b200", "_build", "cugraph.hits.so")
HITS_HOST_SO = os.path.join(REPO, "memgraph_b200", "_build", "libmgp_hits_host.so")
SIGNATURE = ("get(max_iterations = 100 :: INTEGER, tolerance = 1.0000000000000001e-05 :: FLOAT, "
             "normalized = true :: BOOLEAN) :: (node :: NODE, hubs :: FLOAT, authorities :: FLOAT)")

# The engine names a module after its file name without ".so" (cugraph.hits); the in-memory host cuts the name at its
# first dot (cugraph), so an error text starts with either.
PREFIX = r"^cugraph(\.hits)?\.get: "

_host = None


def host():
    global _host
    if _host is None:
        if not os.path.exists(HITS_HOST_SO):
            from memgraph_b200 import build
            build.build_all()
        H = ctypes.CDLL(HITS_HOST_SO, mode=ctypes.RTLD_GLOBAL)
        vp = ctypes.c_void_p
        H.fh_graph_create.restype = vp
        H.fh_graph_create.argtypes = [ctypes.c_uint64, vp, ctypes.c_uint64, vp, vp, ctypes.c_int]
        H.fh_graph_destroy.argtypes = [vp]
        H.fh_graph_set_abort.argtypes = [vp, ctypes.c_int]
        H.fh_graph_hide_vertex.argtypes = [vp, ctypes.c_int64]
        H.fh_live_objects.restype = ctypes.c_long
        H.fh_module_load.restype = vp
        H.fh_module_load.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t]
        H.fh_module_close.argtypes = [vp]
        H.fh_module_signature.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t]
        H.fh_columns_call.restype = vp
        H.fh_columns_call.argtypes = [vp, ctypes.c_char_p, vp, ctypes.c_int, ctypes.c_char_p, vp, vp, ctypes.c_char_p,
                                      ctypes.c_char_p]
        H.fh_columns_result_error.restype = ctypes.c_char_p
        H.fh_columns_result_error.argtypes = [vp]
        H.fh_columns_result_rows.restype = ctypes.c_uint64
        H.fh_columns_result_rows.argtypes = [vp]
        H.fh_columns_result_copy.argtypes = [vp, vp, vp, vp]
        H.fh_columns_result_destroy.argtypes = [vp]
        _host = H
    return _host


class ProcedureError(RuntimeError):
    """What the engine raises as QueryRuntimeException("<module>.<proc>: <msg>")."""


class Graph:
    def __init__(self, gids, src_gid, dst_gid, transactional=True):
        g, s, d = (np.ascontiguousarray(a, dtype=np.int64) for a in (gids, src_gid, dst_gid))
        self.h = host().fh_graph_create(len(g), g.ctypes.data, len(s), s.ctypes.data, d.ctypes.data,
                                        1 if transactional else 0)
        if not self.h:
            raise ValueError("edge endpoint is not a vertex of the graph")

    def hide_vertex(self, gid):
        assert host().fh_graph_hide_vertex(self.h, gid) == 0

    def set_abort(self, flag=True):
        host().fh_graph_set_abort(self.h, 1 if flag else 0)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        host().fh_graph_destroy(self.h)


class Module:
    def __init__(self, path=HITS_MODULE_SO):
        err = ctypes.create_string_buffer(1024)
        self.h = host().fh_module_load(path.encode(), err, 1024)
        if not self.h:
            raise OSError(err.value.decode())

    def signature(self, proc="get"):
        """As the engine prints it; the host keeps a BOOLEAN default as 0 / 1, printed here as false / true."""
        buf = ctypes.create_string_buffer(1024)
        if host().fh_module_signature(self.h, proc.encode(), buf, 1024):
            raise KeyError(proc)
        return buf.value.decode().replace("= 1 :: BOOLEAN", "= true :: BOOLEAN").replace("= 0 :: BOOLEAN",
                                                                                          "= false :: BOOLEAN")

    def call(self, graph, *args, proc="get"):
        """bools are BOOLEAN literals, ints INTEGER, floats FLOAT (strictly typed) -> (node gids, hubs, authorities)."""
        kinds = "".join("b" if isinstance(a, bool) else "i" if isinstance(a, int) else "d" for a in args)
        iv = np.array([int(a) if k in "bi" else 0 for a, k in zip(args, kinds)] + [0], dtype=np.int64)
        dv = np.array([float(a) if k == "d" else 0.0 for a, k in zip(args, kinds)] + [0.0], dtype=np.float64)
        r = host().fh_columns_call(self.h, proc.encode(), graph.h, len(args), kinds.encode(), iv.ctypes.data,
                                   dv.ctypes.data, b"hubs", b"authorities")
        try:
            err = host().fh_columns_result_error(r)
            if err is not None:
                raise ProcedureError(err.decode())
            n = host().fh_columns_result_rows(r)
            nodes, hubs, auth = np.zeros(n, dtype=np.int64), np.zeros(n), np.zeros(n)
            host().fh_columns_result_copy(r, nodes.ctypes.data, hubs.ctypes.data, auth.ctypes.data)
            return nodes, hubs, auth
        finally:
            host().fh_columns_result_destroy(r)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        host().fh_module_close(self.h)


def module_oracle(src, dst, **kw):
    """The module's view: the vertices that occur in an edge, dense in ascending gid."""
    used = sorted(set(int(x) for x in src) | set(int(x) for x in dst))
    dense = {g: i for i, g in enumerate(used)}
    hubs, auth, it, conv = oracle_hits(len(used), [dense[int(x)] for x in src], [dense[int(x)] for x in dst], **kw)
    return np.array(used, dtype=np.int64), hubs, auth


def test_exports_and_imports():
    if not os.path.exists(HITS_MODULE_SO):
        from memgraph_b200 import build
        build.build_all()
    defined = subprocess.run(["nm", "-D", "--defined-only", HITS_MODULE_SO], capture_output=True, text=True,
                             check=True).stdout
    assert " T mgp_init_module" in defined and " T mgp_shutdown_module" in defined
    und = subprocess.run(["nm", "-D", "--undefined-only", HITS_MODULE_SO], capture_output=True, text=True,
                         check=True).stdout
    imported = {line.split()[-1] for line in und.splitlines() if " mgp_" in line}
    header = open(os.path.join(REPO, "include", "mgp_abi.h")).read()
    declared = set(re.findall(r"\b(mgp_[a-z_0-9]+)\s*\(", header))
    assert imported <= declared, imported - declared
    assert {"mgp_value_get_bool", "mgp_type_bool", "mgp_value_make_bool"} <= imported
    assert "cuda" not in und.lower() and "nccl" not in und.lower()


@isolated
def test_signature_is_the_reference_signature():
    with Module() as module:
        assert module.signature() == SIGNATURE


@isolated
def test_argument_errors_and_graphs_that_need_no_device():
    before = host().fh_live_objects()
    with Module() as module:
        with Graph([1, 2, 3], [1, 2], [2, 3]) as g:
            with pytest.raises(ProcedureError, match=r"^'cugraph(\.hits)?\.get' argument named "
                                                     r"'max_iterations' at position 0 must be of type INTEGER\.$"):
                module.call(g, 10.0)
            with pytest.raises(ProcedureError, match=r"'tolerance' at position 1 must be of type FLOAT\.$"):
                module.call(g, 10, 1)
            with pytest.raises(ProcedureError, match=r"'normalized' at position 2 must be of type BOOLEAN\.$"):
                module.call(g, 10, 1e-5, 1)
            with pytest.raises(ProcedureError, match="requires between 0 and 3 arguments"):
                module.call(g, 10, 1e-5, True, 4)
        for gids in ([], [5, 6, 7]):  # the empty graph; vertices without edges: cuGraph knows no vertex, no rows
            with Graph(gids, [], []) as g:
                nodes, hubs, auth = module.call(g)
                assert len(nodes) == len(hubs) == len(auth) == 0
    assert host().fh_live_objects() == before


@isolated
def test_no_device_is_a_loud_procedure_error():
    if conftest.HAVE_GPU:
        return  # this is the no-device behaviour
    with Module() as module, Graph([1, 2], [1], [2]) as g:
        with pytest.raises(ProcedureError, match=PREFIX + "CUDA error"):
            module.call(g)


@pytest.mark.gpu
@isolated
def test_reference_e2e_fixtures_through_the_module():
    with Module() as module:
        for fx in FIXTURES:
            src, dst = [a for a, _ in fx["edges"]], [b for _, b in fx["edges"]]
            with Graph(fx["nodes"], src, dst) as g:
                nodes, hubs, auth = module.call(g, *fx["args"])
            if not fx["nodes"]:
                assert len(nodes) == 0
                continue
            assert nodes.tolist() == sorted(fx["nodes"]), fx["name"]  # ascending gid, one row per vertex in an edge
            dense = {int(g): i for i, g in enumerate(nodes)}
            check_fixture(fx, hubs, auth, dense)
            used, ref_h, ref_a = module_oracle(src, dst)
            assert np.array_equal(used, nodes)
            assert np.allclose(hubs, ref_h, rtol=1e-9, atol=1e-12) and np.allclose(auth, ref_a, rtol=1e-9, atol=1e-12)


@pytest.mark.gpu
@isolated
def test_rows_arguments_and_vanished_vertices():
    rng = np.random.default_rng(21)
    n, m = 500, 4000
    gids = rng.choice(np.arange(20 * n, dtype=np.int64), size=n, replace=False)  # scattered, unsorted
    src, dst = gids[rng.integers(0, n - 20, m)], gids[rng.integers(0, n - 20, m)]  # the last 20 stay isolated
    with Module() as module:
        with Graph(gids, src, dst) as g:
            nodes, hubs, auth = module.call(g, 200, 1e-9, False)
            used, ref_h, ref_a = module_oracle(src, dst, max_iterations=200, tolerance=1e-9, normalized=False)
            assert np.array_equal(nodes, used)  # ascending gid; isolated vertices get no row
            assert np.allclose(hubs, ref_h, rtol=1e-9, atol=1e-12) and np.allclose(auth, ref_a, rtol=1e-9, atol=1e-12)
            assert hubs.max() == 1.0 and auth.max() == 1.0
            nodes, hubs, auth = module.call(g, -1)  # wraps through size_t: runs until it converges
            used, ref_h, ref_a = module_oracle(src, dst, max_iterations=2**64 - 1)
            assert np.allclose(hubs, ref_h, rtol=1e-9, atol=1e-12) and abs(hubs.sum() - 1.0) < 1e-12
            hidden = int(used[7])
            g.hide_vertex(hidden)
            with pytest.raises(ProcedureError, match=PREFIX + "Invalid ID!$"):
                module.call(g)
        with Graph(gids, src, dst, transactional=False) as g:
            g.hide_vertex(hidden)  # still part of the scores, but no row
            nodes, hubs, auth = module.call(g)
            used, ref_h, ref_a = module_oracle(src, dst)
            keep = used != hidden
            assert np.array_equal(nodes, used[keep])
            assert np.allclose(hubs, ref_h[keep], rtol=1e-9, atol=1e-12)
            assert np.allclose(auth, ref_a[keep], rtol=1e-9, atol=1e-12)

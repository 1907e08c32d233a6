"""weakly_connected_components.so (memgraph_b200/csrc/weakly_connected_components_module.cpp) on the in-memory mgp host
with an INTEGER-column call (tests/mgp_wcc_host.cpp).  That host defines the same mgp_* symbols as the other hosts, so
the tests that load it run in a child interpreter (@isolated, tests/_bc_host.py).  No-GPU part: exports and imports,
the registered signature, the empty graph, loud failure without a device.  GPU part (-m gpu): rows as a
gid -> component mapping against the reference module's recorded rows and the oracle on the reference's graph view
(mg_utils.hpp:127-171, mg_graph.hpp:203-240), the e2e fixtures, analytical versus transactional mode."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

import conftest
from _bc_host import REPO, isolated
from test_bc_module import PAGERANK_IMPORTS
from test_wcc_oracle import GOLDEN, oracle_wcc, rows_sha256

WCC_MODULE_SO = os.path.join(REPO, "memgraph_b200", "_build", "weakly_connected_components.so")
WCC_HOST_SO = os.path.join(REPO, "memgraph_b200", "_build", "libmgp_wcc_host.so")
REF_WCC_MODULE_SO = os.path.join(REPO, "oracle", "_ref", "weakly_connected_components_reference.so")
HAVE_REF_MODULE = os.path.exists(REF_WCC_MODULE_SO)
SIGNATURE = "get() :: (node :: NODE, component_id :: INTEGER)"

_host = None


def host():
    global _host
    if _host is None:
        H = ctypes.CDLL(WCC_HOST_SO, mode=ctypes.RTLD_GLOBAL)
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
        H.fh_int_call.restype = vp
        H.fh_int_call.argtypes = [vp, ctypes.c_char_p, vp, ctypes.c_char_p]
        H.fh_int_result_error.restype = ctypes.c_char_p
        H.fh_int_result_error.argtypes = [vp]
        H.fh_int_result_rows.restype = ctypes.c_uint64
        H.fh_int_result_rows.argtypes = [vp]
        H.fh_int_result_copy.argtypes = [vp, vp, vp]
        H.fh_int_result_destroy.argtypes = [vp]
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

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        host().fh_graph_destroy(self.h)


class Module:
    def __init__(self, path):
        err = ctypes.create_string_buffer(1024)
        self.h = host().fh_module_load(path.encode(), err, 1024)
        if not self.h:
            raise OSError(err.value.decode())

    def signature(self, proc="get"):
        buf = ctypes.create_string_buffer(1024)
        if host().fh_module_signature(self.h, proc.encode(), buf, 1024):
            raise KeyError(proc)
        return buf.value.decode()

    def call(self, graph, proc="get", column="component_id"):
        """-> (node gids, the INTEGER column), in the order the module emitted its rows."""
        r = host().fh_int_call(self.h, proc.encode(), graph.h, column.encode())
        try:
            err = host().fh_int_result_error(r)
            if err is not None:
                raise ProcedureError(err.decode())
            n = host().fh_int_result_rows(r)
            nodes, values = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64)
            host().fh_int_result_copy(r, nodes.ctypes.data, values.ctypes.data)
            return nodes, values
        finally:
            host().fh_int_result_destroy(r)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        host().fh_module_close(self.h)


def live_objects():
    return host().fh_live_objects()


def rows_of(nodes, values):
    """The rows as (gid, component) pairs sorted by gid: the reference emits them in an unspecified order."""
    rows = np.stack([np.asarray(nodes, dtype=np.int64), np.asarray(values, dtype=np.int64)], axis=1).reshape(-1, 2)
    rows = rows[np.argsort(rows[:, 0], kind="stable")]
    assert len(np.unique(rows[:, 0])) == len(rows), "a node has two rows"
    return rows


def module_oracle(gids, src, dst, hidden=()):
    """The module's rows on the host's graph view (vertices in ascending gid order), sorted by gid; `hidden` vertices
    keep their component numbers but get no row."""
    order = np.sort(np.asarray(gids, dtype=np.int64))
    index = {int(g): i for i, g in enumerate(order)}
    f = np.array([index[int(s)] for s in src], dtype=np.uint64)
    t = np.array([index[int(d)] for d in dst], dtype=np.uint64)
    comp = oracle_wcc(len(order), f, t)
    keep = ~np.isin(order, np.asarray(list(hidden), dtype=np.int64))
    return np.stack([order[keep], comp[keep]], axis=1).reshape(-1, 2)


def wcc_scattered_graphs():
    """(name, gids, src, dst) of tests/golden/wcc_ref_module_rows.json: non-contiguous unsorted gids; random edges with
    multi-edges, self-loops and isolated vertices; one graph whose first vertex's component is not the largest."""
    rng = np.random.default_rng(20261016)
    out = []
    for name, n, m in [("sparse", 300, 150), ("medium", 500, 450), ("dense", 400, 1600)]:
        gids = rng.choice(np.arange(10 * n + 7, dtype=np.int64), size=n, replace=False)
        src, dst = gids[rng.integers(0, n, m)], gids[rng.integers(0, n, m)]
        src = np.concatenate([src, src[:5], gids[:3]])  # multi-edges and self-loops for certain
        dst = np.concatenate([dst, dst[:5], gids[:3]])
        out.append((name, gids, src, dst))
    # the smallest gid sits in a 2-vertex component, the largest component (a 40-vertex path) comes later
    gids = np.arange(1000, 1000 + 60 * 3, 3, dtype=np.int64)
    src = np.concatenate([[gids[0]], gids[10:49]])
    dst = np.concatenate([[gids[1]], gids[11:50]])
    out.append(("first_not_largest", gids[::-1].copy(), src, dst))
    return out


def recorded_rows():
    return json.load(open(os.path.join(GOLDEN, "wcc_ref_module_rows.json")))


def check_e2e_fixtures(module):
    for case in json.load(open(os.path.join(GOLDEN, "wcc_e2e_cases.json")))["cases"]:
        for step in case["steps"]:
            nodes = step["nodes"]
            gids = [100 + 7 * i for i in range(len(nodes))]
            gid_of = dict(zip(nodes, gids))
            with Graph(gids, [gid_of[a] for a, _ in step["edges"]], [gid_of[b] for _, b in step["edges"]]) as g:
                got_nodes, got_values = module.call(g)
            rows = sorted((nodes[gids.index(int(gid))], int(c)) for gid, c in zip(got_nodes, got_values))
            assert rows == [(o["node_id"], o["component_id"]) for o in step["output"]], case["name"]


def test_exports_and_imports():
    if not os.path.exists(WCC_MODULE_SO):
        from memgraph_b200 import build
        build.build_all()
    out = subprocess.run(["nm", "-D", "--defined-only", WCC_MODULE_SO], capture_output=True, text=True,
                         check=True).stdout
    assert " T mgp_init_module" in out and " T mgp_shutdown_module" in out
    und = subprocess.run(["nm", "-D", "--undefined-only", WCC_MODULE_SO], capture_output=True, text=True,
                         check=True).stdout
    strong = {line.split()[-1] for line in und.splitlines() if " U mgp_" in line}
    assert strong <= PAGERANK_IMPORTS, strong - PAGERANK_IMPORTS
    assert "cuda" not in und.lower() and "nccl" not in und.lower()


@isolated
def test_signature_is_the_reference_signature():
    with Module(WCC_MODULE_SO) as module:
        sig = module.signature()
    assert sig == SIGNATURE
    assert recorded_rows()["signature"] == SIGNATURE
    if HAVE_REF_MODULE:
        with Module(REF_WCC_MODULE_SO) as ref:
            assert ref.signature() == sig


@isolated
def test_empty_graph_and_no_device():
    before = live_objects()
    with Module(WCC_MODULE_SO) as module:
        with Graph([], [], []) as g:
            nodes, values = module.call(g)
            assert len(nodes) == 0 and len(values) == 0
        if not conftest.HAVE_GPU:
            with Graph([5, 9, 2], [5, 9], [9, 2]) as g:
                with pytest.raises(ProcedureError, match=r"^weakly_connected_components\.get: CUDA error"):
                    module.call(g)
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_rows_equal_the_reference_rows_and_the_oracle():
    before = live_objects()
    with Module(WCC_MODULE_SO) as module:
        for (name, gids, src, dst), call in zip(wcc_scattered_graphs(), recorded_rows()["graphs"]):
            with Graph(gids, src, dst) as g:
                nodes, values = module.call(g)
            assert np.array_equal(nodes, np.sort(gids)), name  # rows come in dense order here
            rows = rows_of(nodes, values)
            assert rows_sha256(rows) == call["rows_sha256"], name
            assert np.array_equal(rows, module_oracle(gids, src, dst)), name
        check_e2e_fixtures(module)
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_analytical_and_transactional_mode():
    gids = np.array([30, 10, 20, 70, 50, 90, 80], dtype=np.int64)
    src, dst = np.array([30, 70, 90]), np.array([10, 50, 80])
    with Module(WCC_MODULE_SO) as module:
        with Graph(gids, src, dst) as g:
            assert np.array_equal(rows_of(*module.call(g)), module_oracle(gids, src, dst))
            g.hide_vertex(20)
            with pytest.raises(ProcedureError, match=r"^weakly_connected_components\.get: Invalid ID!$"):
                module.call(g)
        with Graph(gids, src, dst, transactional=False) as g:
            g.hide_vertex(20)  # its own component: number 1 stays used, the next component is still 2
            rows = rows_of(*module.call(g))
            assert np.array_equal(rows, module_oracle(gids, src, dst, hidden=[20]))
            assert rows[:, 1].tolist() == [0, 0, 2, 2, 3, 3]

"""bridges.so and biconnected_components.so (memgraph_b200/csrc/biconnectivity_modules.cpp) on the in-memory mgp host
with edge rows (tests/mgp_edge_host.cpp).  That host defines the same mgp_* symbols as the other hosts, so the tests that
load it run in a child interpreter (@isolated, tests/_bc_host.py).  No-GPU part: exports and imports, the registered
signatures against the recorded reference signatures, the empty graph, loud failure without a device.  GPU part
(-m gpu): rows against the reference modules' recorded rows and the oracle on the reference's graph view
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
from test_biconnectivity_oracle import GOLDEN, bcc_partition, oracle_biconnectivity

BUILD = os.path.join(REPO, "memgraph_b200", "_build")
MODULE_SO = {"bridges": os.path.join(BUILD, "bridges.so"),
             "biconnected_components": os.path.join(BUILD, "biconnected_components.so")}
REF_MODULE_SO = {name: os.path.join(REPO, "oracle", "_ref", f"{name}_reference.so") for name in MODULE_SO}
HAVE_REF_MODULES = all(os.path.exists(p) for p in REF_MODULE_SO.values())
EDGE_HOST_SO = os.path.join(BUILD, "libmgp_edge_host.so")
SIGNATURE = {"bridges": "get() :: (node_from :: NODE, node_to :: NODE)",
             "biconnected_components": "get() :: (bcc_id :: INTEGER, node_from :: NODE, node_to :: NODE)"}

_host = None


def host():
    global _host
    if _host is None:
        H = ctypes.CDLL(EDGE_HOST_SO, mode=ctypes.RTLD_GLOBAL)
        vp = ctypes.c_void_p
        H.fh_graph_create.restype = vp
        H.fh_graph_create.argtypes = [ctypes.c_uint64, vp, ctypes.c_uint64, vp, vp, ctypes.c_int]
        H.fh_graph_destroy.argtypes = [vp]
        H.fh_graph_hide_vertex.argtypes = [vp, ctypes.c_int64]
        H.fh_live_objects.restype = ctypes.c_long
        H.fh_module_load.restype = vp
        H.fh_module_load.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t]
        H.fh_module_close.argtypes = [vp]
        H.fh_module_signature.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t]
        H.fh_edge_call.restype = vp
        H.fh_edge_call.argtypes = [vp, ctypes.c_char_p, vp, ctypes.c_char_p]
        H.fh_edge_result_error.restype = ctypes.c_char_p
        H.fh_edge_result_error.argtypes = [vp]
        H.fh_edge_result_rows.restype = ctypes.c_uint64
        H.fh_edge_result_rows.argtypes = [vp]
        H.fh_edge_result_copy.argtypes = [vp, vp, vp, vp]
        H.fh_edge_result_destroy.argtypes = [vp]
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

    def call(self, graph, proc="get"):
        """-> int64[rows, 3]: (bcc_id or 0, node_from gid, node_to gid), in the order the module emitted its rows."""
        r = host().fh_edge_call(self.h, proc.encode(), graph.h, b"bcc_id")
        try:
            err = host().fh_edge_result_error(r)
            if err is not None:
                raise ProcedureError(err.decode())
            n = host().fh_edge_result_rows(r)
            rows = [np.zeros(n, dtype=np.int64) for _ in range(3)]
            host().fh_edge_result_copy(r, *(a.ctypes.data for a in rows))
            return np.stack(rows, axis=1).reshape(-1, 3)
        finally:
            host().fh_edge_result_destroy(r)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        host().fh_module_close(self.h)


def live_objects():
    return host().fh_live_objects()


def view_coo(gids, src, dst):
    """The host's graph view: vertices in ascending gid order, out-edges grouped by source in insertion order.
    -> (sorted gids, dense from, dense to, gid from, gid to), edges in view order."""
    order = np.sort(np.asarray(gids, dtype=np.int64))
    index = {int(g): i for i, g in enumerate(order)}
    f = np.array([index[int(s)] for s in src], dtype=np.uint64)
    t = np.array([index[int(d)] for d in dst], dtype=np.uint64)
    perm = np.argsort(f, kind="stable")
    f, t = f[perm], t[perm]
    return order, f, t, order[f.astype(np.int64)], order[t.astype(np.int64)]


def module_oracle(name, gids, src, dst, hidden=()):
    """The rows our module must emit, in its order: bridges in view edge order; components grouped by ascending bcc_id
    (first-edge numbering), view edge order inside.  Rows touching a `hidden` vertex are skipped."""
    order, f, t, gf, gt = view_coo(gids, src, dst)
    bridge, bcc = oracle_biconnectivity(len(order), f, t)
    keep = ~(np.isin(gf, list(hidden)) | np.isin(gt, list(hidden)))
    if name == "bridges":
        sel = (bridge == 1) & keep
        return np.stack([np.zeros(sel.sum(), dtype=np.int64), gf[sel], gt[sel]], axis=1).reshape(-1, 3)
    sel = (bcc >= 0) & keep
    idx = np.nonzero(sel)[0]
    idx = idx[np.argsort(bcc[idx], kind="stable")]
    return np.stack([bcc[idx], gf[idx], gt[idx]], axis=1).reshape(-1, 3)


def same_bridges(a, b):
    """Equal sets of (from, to)."""
    return {(int(x), int(y)) for _, x, y in a} == {(int(x), int(y)) for _, x, y in b}


def same_components(ref_rows, rows):
    """Equal partitions of distinct unordered non-loop pairs under a bijection of ids; the reference may drop parallel
    copies of tree edges, so its row count is at most ours."""
    return len(ref_rows) <= len(rows) and bcc_partition(ref_rows) == bcc_partition(rows)


def scattered_graphs():
    """(name, gids, src, dst) of tests/golden/biconnectivity_ref_module_rows.json: non-contiguous unsorted gids;
    multi-edges, self-loops, isolated vertices and several components; sparse graphs so that blocks and bridges mix."""
    rng = np.random.default_rng(20261017)
    out = []
    for name, n, m in [("forest", 200, 150), ("sparse", 300, 330), ("medium", 400, 600), ("dense", 150, 900)]:
        gids = rng.choice(np.arange(10 * n + 7, dtype=np.int64), size=n, replace=False)
        src, dst = gids[rng.integers(0, n, m)], gids[rng.integers(0, n, m)]
        src = np.concatenate([src, src[:6], gids[:3], dst[6:9]])  # multi-edges both ways and self-loops for certain
        dst = np.concatenate([dst, dst[:6], gids[:3], src[6:9]])
        out.append((name, gids, src, dst))
    # cycles joined by bridges, with a doubled tree edge and an isolated vertex
    gids = np.arange(5000, 5000 + 40 * 7, 7, dtype=np.int64)
    pairs = [(0, 1), (1, 2), (2, 0), (2, 3), (3, 4), (4, 5), (5, 3), (5, 6), (6, 7), (6, 7), (7, 8), (8, 9), (9, 7),
             (10, 11), (11, 12), (12, 13), (13, 10), (13, 14), (14, 14), (15, 16)]
    out.append(("cycles_and_bridges", gids[::-1].copy(), gids[[a for a, _ in pairs]], gids[[b for _, b in pairs]]))
    return out


def recorded_rows():
    return json.load(open(os.path.join(GOLDEN, "biconnectivity_ref_module_rows.json")))


def e2e_cases():
    return json.load(open(os.path.join(GOLDEN, "biconnectivity_e2e_cases.json")))["cases"]


def check_e2e_fixtures(modules):
    """modules: name -> Module.  The e2e queries sort their rows, so (component, from, to) tuples compare directly for
    bridges; component ids compare as partitions."""
    for case in e2e_cases():
        nodes = case["nodes"]
        gids = [100 + 7 * i for i in range(len(nodes))]
        gid_of = dict(zip(nodes, gids))
        node_of = dict(zip(gids, nodes))
        with Graph(gids, [gid_of[a] for a, _ in case["edges"]], [gid_of[b] for _, b in case["edges"]]) as g:
            rows = modules[case["module"]].call(g)
        got = [(int(c), node_of[int(a)], node_of[int(b)]) for c, a, b in rows]
        if case["module"] == "bridges":
            assert sorted((a, b) for _, a, b in got) == [(o["from_id"], o["to_id"]) for o in case["output"]], case["name"]
        else:
            exp = [(o["component"], o["from_id"], o["to_id"]) for o in case["output"]]
            assert bcc_partition(exp) == bcc_partition(got) and len(exp) == len(got), case["name"]


def test_exports_and_imports():
    for path in MODULE_SO.values():
        if not os.path.exists(path):
            from memgraph_b200 import build
            build.build_all()
        out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
        assert " T mgp_init_module" in out and " T mgp_shutdown_module" in out
        und = subprocess.run(["nm", "-D", "--undefined-only", path], capture_output=True, text=True, check=True).stdout
        strong = {line.split()[-1] for line in und.splitlines() if " U mgp_" in line}
        assert strong <= PAGERANK_IMPORTS, strong - PAGERANK_IMPORTS
        assert "cuda" not in und.lower() and "nccl" not in und.lower()


@isolated
def test_signatures_are_the_reference_signatures():
    recorded = recorded_rows()["modules"]
    for name, path in MODULE_SO.items():
        with Module(path) as module:
            sig = module.signature()
        assert sig == SIGNATURE[name] == recorded[name]["signature"], name
        if HAVE_REF_MODULES:
            with Module(REF_MODULE_SO[name]) as ref:
                assert ref.signature() == sig, name


@isolated
def test_empty_graph_and_no_device():
    before = live_objects()
    for name, path in MODULE_SO.items():
        with Module(path) as module:
            with Graph([], [], []) as g:
                assert len(module.call(g)) == 0
            if not conftest.HAVE_GPU:
                with Graph([5, 9, 2], [5, 9], [9, 2]) as g:
                    with pytest.raises(ProcedureError, match=rf"^{name}\.get: CUDA error"):
                        module.call(g)
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_rows_equal_the_reference_rows_and_the_oracle():
    before = live_objects()
    recorded = recorded_rows()["modules"]
    modules = {name: Module(path) for name, path in MODULE_SO.items()}
    try:
        for name, module in modules.items():
            graphs = recorded[name]["graphs"]
            assert [c["name"] for c in graphs] == [g[0] for g in scattered_graphs()]
            for (gname, gids, src, dst), call in zip(scattered_graphs(), graphs):
                with Graph(gids, src, dst) as g:
                    rows = module.call(g)
                assert np.array_equal(rows, module_oracle(name, gids, src, dst)), (name, gname)
                ref = np.array(call["rows"], dtype=np.int64).reshape(-1, 3)
                if name == "bridges":
                    assert same_bridges(ref, rows), gname
                else:
                    assert same_components(ref, rows), gname
        check_e2e_fixtures(modules)
    finally:
        for module in modules.values():
            module.__exit__()
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_analytical_and_transactional_mode():
    gids = np.array([30, 10, 20, 70, 50, 90, 80], dtype=np.int64)
    src = np.array([10, 20, 30, 30, 50, 70, 90])
    dst = np.array([20, 30, 10, 50, 70, 80, 80])  # triangle 10-20-30, path 30-50-70-80, bridge 90-80
    for name, path in MODULE_SO.items():
        with Module(path) as module:
            with Graph(gids, src, dst) as g:
                assert np.array_equal(module.call(g), module_oracle(name, gids, src, dst)), name
                g.hide_vertex(50)
                with pytest.raises(ProcedureError, match=rf"^{name}\.get: Invalid ID!$"):
                    module.call(g)
            with Graph(gids, src, dst, transactional=False) as g:
                g.hide_vertex(50)  # its edges get no row; the components' numbers stay as computed with it
                rows = module.call(g)
                assert np.array_equal(rows, module_oracle(name, gids, src, dst, hidden=[50])), name
                assert 50 not in rows[:, 1:]

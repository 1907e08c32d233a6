"""gpu_wsp.so (memgraph_b200/csrc/gpu_wsp_module.cpp) on the in-memory mgp host with a node / FLOAT / INTEGER call and a
STRING edge property (tests/mgp_wsp_host.cpp).  That host defines the same mgp_* symbols as the other hosts, so every
test that loads it runs in a child interpreter (@isolated, tests/_bc_host.py).  No-GPU part: exports and imports, the
registered signature, argument errors, abort, loud failure without a device.  GPU part (-m gpu): the reference's
fixtures, integer and float properties, the engine's error texts and which edges are checked."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

import conftest
from _bc_host import REPO, isolated
from test_bc_module import PAGERANK_IMPORTS
from test_wsp_oracle import fixture_cases, oracle_wsp

WSP_MODULE_SO = os.path.join(REPO, "memgraph_b200", "_build", "gpu_wsp.so")
WSP_HOST_SO = os.path.join(REPO, "memgraph_b200", "_build", "libmgp_wsp_host.so")
SIGNATURE = ("distances(source :: NODE, weight_property = \"weight\" :: STRING, direction = 0 :: INTEGER, "
             "upper_bound = -1 :: INTEGER) :: (node :: NODE, total_weight :: FLOAT, hops :: INTEGER)")
# the host's tagged properties (tests/mgp_wsp_host.cpp): a STRING, a DOUBLE NaN and a DURATION
STRING_WEIGHT, NAN_WEIGHT, DURATION_WEIGHT = np.array([0x7FF8000053545200, 0x7FF800004E414E00, 0x7FF8000044555200],
                                                      dtype=np.uint64).view(np.float64)
DEPTH_MESSAGE = "Maximum depth in weighted shortest path expansion must be at least 1."
NULL_MESSAGE = ("All weights should be of the same type, either numeric or a Duration. Please update the weight "
                "expression or the filter expression. For more details, visit https://memgr.ph/wsp.")

_host = None


def host():
    global _host
    if _host is None:
        H = ctypes.CDLL(WSP_HOST_SO, mode=ctypes.RTLD_GLOBAL)
        vp = ctypes.c_void_p
        H.fh_graph_create.restype = vp
        H.fh_graph_create.argtypes = [ctypes.c_uint64, vp, ctypes.c_uint64, vp, vp, ctypes.c_int]
        H.fh_graph_destroy.argtypes = [vp]
        H.fh_graph_set_edge_property.argtypes = [vp, ctypes.c_char_p, ctypes.c_uint64, vp, vp, ctypes.c_int]
        H.fh_graph_set_abort.argtypes = [vp, ctypes.c_int]
        H.fh_graph_hide_vertex.argtypes = [vp, ctypes.c_int64]
        H.fh_live_objects.restype = ctypes.c_long
        H.fh_module_load.restype = vp
        H.fh_module_load.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t]
        H.fh_module_close.argtypes = [vp]
        H.fh_module_signature.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t]
        H.fh_wsp_call.restype = vp
        H.fh_wsp_call.argtypes = [vp, ctypes.c_char_p, vp, ctypes.c_int, ctypes.c_char_p, vp, vp, vp, ctypes.c_char_p,
                                  ctypes.c_char_p]
        H.fh_wsp_result_error.restype = ctypes.c_char_p
        H.fh_wsp_result_error.argtypes = [vp]
        H.fh_wsp_result_rows.restype = ctypes.c_uint64
        H.fh_wsp_result_rows.argtypes = [vp]
        H.fh_wsp_result_copy.argtypes = [vp, vp, vp, vp]
        H.fh_wsp_result_destroy.argtypes = [vp]
        _host = H
    return _host


class ProcedureError(RuntimeError):
    """What the engine raises as QueryRuntimeException("<module>.<proc>: <msg>")."""


class Node:
    def __init__(self, gid):
        self.gid = int(gid)


class Graph:
    """gids, edges as gid pairs, and optionally one numeric edge property per edge (NaN = absent)."""

    def __init__(self, gids, src, dst, weights=None, name="weight", as_int=False, transactional=True):
        g, s, d = (np.ascontiguousarray(a, dtype=np.int64) for a in (gids, src, dst))
        self.h = host().fh_graph_create(len(g), g.ctypes.data, len(s), s.ctypes.data, d.ctypes.data,
                                        1 if transactional else 0)
        if not self.h:
            raise ValueError("edge endpoint is not a vertex of the graph")
        if weights is not None:
            w = np.ascontiguousarray(weights, dtype=np.float64)
            assert host().fh_graph_set_edge_property(self.h, name.encode(), len(w), s.ctypes.data, w.ctypes.data,
                                                     1 if as_int else 0) == 0

    def set_abort(self, flag=True):
        host().fh_graph_set_abort(self.h, 1 if flag else 0)

    def hide_vertex(self, gid):
        assert host().fh_graph_hide_vertex(self.h, gid) == 0

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        host().fh_graph_destroy(self.h)


class Module:
    def __init__(self, path=WSP_MODULE_SO):
        err = ctypes.create_string_buffer(1024)
        self.h = host().fh_module_load(path.encode(), err, 1024)
        if not self.h:
            raise OSError(err.value.decode())

    def signature(self, proc="distances"):
        buf = ctypes.create_string_buffer(1024)
        if host().fh_module_signature(self.h, proc.encode(), buf, 1024):
            raise KeyError(proc)
        return buf.value.decode()

    def call(self, graph, *args, proc="distances"):
        """Node -> NODE, str -> STRING, int -> INTEGER, float -> FLOAT.  -> (node gids, total_weight, hops)."""
        kinds = "".join("v" if isinstance(a, Node) else "s" if isinstance(a, str) else "i" if isinstance(a, int)
                        else "d" for a in args)
        iv = np.array([a.gid if k == "v" else int(a) if k == "i" else 0 for a, k in zip(args, kinds)] + [0],
                      dtype=np.int64)
        dv = np.array([float(a) if k == "d" else 0.0 for a, k in zip(args, kinds)] + [0.0], dtype=np.float64)
        sv = (ctypes.c_char_p * (len(args) + 1))(*[a.encode() if k == "s" else None for a, k in zip(args, kinds)], None)
        r = host().fh_wsp_call(self.h, proc.encode(), graph.h, len(args), kinds.encode(), iv.ctypes.data,
                               dv.ctypes.data, sv, b"total_weight", b"hops")
        try:
            err = host().fh_wsp_result_error(r)
            if err is not None:
                raise ProcedureError(err.decode())
            n = host().fh_wsp_result_rows(r)
            nodes, totals, hops = np.zeros(n, dtype=np.int64), np.zeros(n), np.zeros(n, dtype=np.int64)
            host().fh_wsp_result_copy(r, nodes.ctypes.data, totals.ctypes.data, hops.ctypes.data)
            return nodes, totals, hops
        finally:
            host().fh_wsp_result_destroy(r)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        host().fh_module_close(self.h)


def live_objects():
    return host().fh_live_objects()


def fixture_graph(case):
    """(gids, Graph) for a fixture: dense id i has gid 100 + 7 i; an all-INTEGER case hands out INTEGER values."""
    gids = [100 + 7 * i for i in range(case["n"])]
    src = [gids[a] for a, *_ in case["edges"]]
    dst = [gids[b] for _, b, *_ in case["edges"]]
    w = [STRING_WEIGHT if ty == "string" else float(x) for *_, x, ty in case["edges"]]
    as_int = all(ty in ("int", "string") for *_, ty in case["edges"])
    return gids, Graph(gids, src, dst, w, as_int=as_int)


def test_exports_and_imports():
    if not os.path.exists(WSP_MODULE_SO) or not os.path.exists(WSP_HOST_SO):
        from memgraph_b200 import build
        build.build_all()
    out = subprocess.run(["nm", "-D", "--defined-only", WSP_MODULE_SO], capture_output=True, text=True,
                         check=True).stdout
    assert " T mgp_init_module" in out and " T mgp_shutdown_module" in out
    und = subprocess.run(["nm", "-D", "--undefined-only", WSP_MODULE_SO], capture_output=True, text=True,
                         check=True).stdout
    strong = {line.split()[-1] for line in und.splitlines() if " U mgp_" in line}
    extra = {"mgp_edge_get_property", "mgp_value_get_type", "mgp_type_string", "mgp_value_get_string",
             "mgp_value_make_string", "mgp_value_get_vertex", "mgp_proc_add_arg"}
    assert strong <= PAGERANK_IMPORTS | extra, strong - PAGERANK_IMPORTS - extra
    assert "cuda" not in und.lower() and "nccl" not in und.lower()


@isolated
def test_signature_and_defaults():
    with Module() as module:
        assert module.signature() == SIGNATURE
        with Graph([1, 2], [1], [2], [1.0]) as g:
            with pytest.raises(ProcedureError, match=r"must be of type STRING"):
                module.call(g, Node(1), 3)
            with pytest.raises(ProcedureError, match=r"must be of type INTEGER"):
                module.call(g, Node(1), "weight", 0.5)
            with pytest.raises(ProcedureError, match=r"requires between 1 and 4 arguments"):
                module.call(g)


@isolated
def test_upper_bound_below_one_and_bad_direction_are_errors():
    before = live_objects()
    with Module() as module, Graph([1, 2], [1], [2], [1.0]) as g:
        for ub in (0, -2, -100):
            with pytest.raises(ProcedureError, match="^gpu_wsp.distances: " + DEPTH_MESSAGE + "$"):
                module.call(g, Node(1), "weight", 0, ub)
        with pytest.raises(ProcedureError, match=r"direction must be 0 \(OUT\), 1 \(IN\) or 2 \(BOTH\)"):
            module.call(g, Node(1), "weight", 3)
    assert live_objects() == before


@isolated
def test_abort_and_no_device():
    before = live_objects()
    with Module() as module:
        with Graph([5, 9, 2], [5, 9], [9, 2], [1.0, 2.0]) as g:
            g.set_abort(True)
            with pytest.raises(ProcedureError, match=r"^gpu_wsp\.distances: procedure aborted by the host$"):
                module.call(g, Node(5))
            g.set_abort(False)
            if not conftest.HAVE_GPU:
                with pytest.raises(ProcedureError, match=r"^gpu_wsp\.distances: CUDA error"):
                    module.call(g, Node(5))
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_reference_fixtures_through_the_module():
    before = live_objects()
    with Module() as module:
        for case in fixture_cases():
            gids, graph = fixture_graph(case)
            ub = -1 if case["upper_bound"] is None else case["upper_bound"]
            if "error" in case and case["error"]["kind"] == "upper_bound":
                ub = -2  # -1 is the procedure's "unbounded"; every other value below 1 raises the engine's text
            with graph as g:
                if "error" in case:
                    with pytest.raises(ProcedureError) as err:
                        module.call(g, Node(gids[case["start"]]), "weight", case["direction"], ub)
                    assert str(err.value) == "gpu_wsp.distances: " + case["error"]["message"], case["name"]
                    continue
                nodes, totals, hops = module.call(g, Node(gids[case["start"]]), "weight", case["direction"], ub)
            expected = sorted(case["rows"])  # rows come in dense order here
            assert nodes.tolist() == [gids[v] for v, *_ in expected], case["name"]
            assert totals.tolist() == [float(t) for _, t, _ in expected], case["name"]
            for h, (_, _, size) in zip(hops.tolist(), expected):
                assert size is None or h == size, case["name"]
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_integer_and_float_properties_and_the_oracle():
    rng = np.random.default_rng(5)
    with Module() as module:
        for trial in range(12):
            n, m = 60, 200
            gids = rng.choice(np.arange(10 * n), size=n, replace=False)
            f, t = rng.integers(0, n, m), rng.integers(0, n, m)
            as_int = trial % 2 == 0
            w = rng.integers(0, 17, m).astype(np.float64) if as_int else rng.random(m)
            direction, ub = trial % 3, [-1, 1, 2, 3][trial % 4]
            order = np.argsort(gids)  # the host iterates vertices in ascending gid order: that is the dense order
            dense = np.empty(n, dtype=np.int64)
            dense[order] = np.arange(n)
            with Graph(gids, gids[f], gids[t], w, as_int=as_int) as g:
                nodes, totals, hops = module.call(g, Node(gids[0]), "weight", direction, ub)
            # the module's edge list is the host's out-edge order: sources ascending by gid, then insertion order
            edge_order = np.argsort(dense[f], kind="stable")
            rc, dist, _, ohops, _ = oracle_wsp(n, dense[f][edge_order], dense[t][edge_order], w[edge_order],
                                              dense[0], direction, None if ub == -1 else ub)
            assert rc == 0
            produced = np.flatnonzero(~np.isnan(dist))
            assert nodes.tolist() == np.sort(gids)[produced].tolist(), trial
            assert totals.tobytes() == dist[produced].tobytes(), trial
            assert hops.tolist() == ohops[produced].tolist(), trial


@pytest.mark.gpu
@isolated
def test_error_texts_and_which_edges_are_checked():
    before = live_objects()
    with Module() as module:
        # a path 1 -> 2 -> 3 -> 4; the bad weight sits on 3 -> 4
        gids, src, dst = [1, 2, 3, 4, 5], [1, 2, 3, 5], [2, 3, 4, 1]
        for bad, message in [(STRING_WEIGHT, "Weight must be numeric or a Duration, got string."),
                             (-10.0, "Weight must be non-negative, got -10."),
                             (-0.5, "Weight must be non-negative, got -0.5."),
                             (-1e20, "Weight must be non-negative, got -1e+20."),
                             (-1.5e-7, "Weight must be non-negative, got -1.5e-07."),
                             (-1e-5, "Weight must be non-negative, got -1e-05."),
                             (-2.5e-5, "Weight must be non-negative, got -2.5e-05."),
                             (-1e-4, "Weight must be non-negative, got -0.0001."),
                             (-1e15, "Weight must be non-negative, got -1000000000000000."),
                             (-1e16, "Weight must be non-negative, got -1e+16."),
                             (-123456.789, "Weight must be non-negative, got -123456.789."),
                             (NAN_WEIGHT, "Weight must not be NaN."),
                             (DURATION_WEIGHT, "Duration weights are not supported by gpu_wsp."),
                             (math.nan, NULL_MESSAGE)]:
            with Graph(gids, src, dst, [1.0, 2.0, bad, 1.0]) as g:
                with pytest.raises(ProcedureError) as err:
                    module.call(g, Node(1))
                assert str(err.value) == "gpu_wsp.distances: " + message
                # vertex 3 sits at depth 2 == upper_bound: it is not expanded, so its edge is never evaluated
                nodes, totals, hops = module.call(g, Node(1), "weight", 0, 2)
                assert nodes.tolist() == [2, 3] and totals.tolist() == [1.0, 3.0] and hops.tolist() == [1, 2]
                # the bad edge is unreachable from 4 and from 2 walking IN
                assert module.call(g, Node(4))[0].tolist() == []
                assert module.call(g, Node(2), "weight", 1)[0].tolist() == [1, 5]
        # the smallest pulled edge among the evaluated bad ones is quoted: vertex 1's edges come first
        with Graph([1, 2, 3], [1, 1, 2], [2, 3, 3], [-2.0, STRING_WEIGHT, -3.0]) as g:
            with pytest.raises(ProcedureError, match=r"got -2\.$"):
                module.call(g, Node(1))
        # an absent property is the engine's null-weight text; another property name reads as absent everywhere
        with Graph([1, 2], [1], [2], [1.0]) as g:
            with pytest.raises(ProcedureError, match="All weights should be of the same type"):
                module.call(g, Node(1), "cost")
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_analytical_mode_and_infinite_weights():
    with Module() as module:
        with Graph([1, 2, 3], [1, 2], [2, 3], [math.inf, 0.0]) as g:
            nodes, totals, hops = module.call(g, Node(1))
            assert nodes.tolist() == [2, 3] and totals.tolist() == [math.inf, math.inf] and hops.tolist() == [1, 2]
            g.hide_vertex(3)
            with pytest.raises(ProcedureError, match=r"^gpu_wsp\.distances: Invalid ID!$"):
                module.call(g, Node(1))
        with Graph([1, 2, 3], [1, 2], [2, 3], [1.0, 2.0], transactional=False) as g:
            g.hide_vertex(2)
            nodes, totals, _ = module.call(g, Node(1))
            assert nodes.tolist() == [3] and totals.tolist() == [3.0]

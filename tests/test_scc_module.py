"""strongly_connected_components.so (memgraph_b200/csrc/strongly_connected_components_module.cpp) on the in-memory mgp
host with an INTEGER-column call (tests/mgp_wcc_host.cpp; child interpreters as in tests/test_wcc_module.py).  No-GPU
part: exports and imports, the registered signature, zero rows for an empty graph, loud failure without a device, the
host's abort flag.  GPU part (-m gpu): rows as a gid -> component mapping against the oracle on the module's graph view,
analytical versus transactional mode with a hidden vertex."""
import os
import subprocess

import numpy as np
import pytest

import conftest
from _bc_host import REPO, isolated
from test_bc_module import PAGERANK_IMPORTS
from test_scc_oracle import golden, handmade_graphs, oracle_scc, seeded_graphs
from test_wcc_module import Graph, Module, ProcedureError, host, live_objects, rows_of

MODULE_SO = os.path.join(REPO, "memgraph_b200", "_build", "strongly_connected_components.so")
SIGNATURE = "get() :: (node :: NODE, component_id :: INTEGER)"


def module_oracle(gids, src, dst, hidden=()):
    """The module's rows on the host's graph view (vertices in ascending gid order), sorted by gid; `hidden` vertices
    keep their component numbers but get no row."""
    order = np.sort(np.asarray(gids, dtype=np.int64))
    dense = np.searchsorted(order, np.asarray(src, dtype=np.int64)), np.searchsorted(order, np.asarray(dst, dtype=np.int64))
    comp = oracle_scc(len(order), dense[0], dense[1])
    keep = ~np.isin(order, np.asarray(list(hidden), dtype=np.int64))
    return np.stack([order[keep], comp[keep]], axis=1).reshape(-1, 2)


def test_exports_and_imports():
    if not os.path.exists(MODULE_SO):
        from memgraph_b200 import build
        build.build_all()
    out = subprocess.run(["nm", "-D", "--defined-only", MODULE_SO], capture_output=True, text=True, check=True).stdout
    assert " T mgp_init_module" in out and " T mgp_shutdown_module" in out
    und = subprocess.run(["nm", "-D", "--undefined-only", MODULE_SO], capture_output=True, text=True,
                         check=True).stdout
    strong = {line.split()[-1] for line in und.splitlines() if " U mgp_" in line}
    assert strong <= PAGERANK_IMPORTS, strong - PAGERANK_IMPORTS
    assert "cuda" not in und.lower() and "nccl" not in und.lower()


@isolated
def test_signature():
    with Module(MODULE_SO) as module:
        assert module.signature() == SIGNATURE


@isolated
def test_empty_graph_no_device_and_abort():
    before = live_objects()
    with Module(MODULE_SO) as module:
        with Graph([], [], []) as g:
            nodes, values = module.call(g)
            assert len(nodes) == 0 and len(values) == 0
        if not conftest.HAVE_GPU:
            with Graph([5, 9, 2], [5, 9], [9, 2]) as g:
                with pytest.raises(ProcedureError, match=r"^strongly_connected_components\.get: CUDA error"):
                    module.call(g)
        with Graph([5, 9, 2], [5, 9, 2], [9, 2, 5]) as g:
            host().fh_graph_set_abort(g.h, 1)
            with pytest.raises(ProcedureError,
                               match=r"^strongly_connected_components\.get: procedure aborted by the host$"):
                module.call(g)
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_rows_equal_the_oracle():
    before = live_objects()
    rng = np.random.default_rng(41)
    graphs = [(n, [a for a, _ in e], [b for _, b in e]) for _, n, e in handmade_graphs()]
    graphs += [(n, f, t) for _, n, f, t in seeded_graphs()]
    recorded = [c["components"] for c in golden()["handmade"] + golden()["seeded"]]
    with Module(MODULE_SO) as module:
        for (n, f, t), expected in zip(graphs, recorded):
            gids = np.sort(rng.choice(np.arange(20 * n + 5, dtype=np.int64), size=n, replace=False))
            scattered = rng.permutation(gids)  # created out of order; the host visits them in gid order
            src, dst = gids[np.asarray(f, dtype=np.int64)], gids[np.asarray(t, dtype=np.int64)]
            with Graph(scattered, src, dst) as g:
                nodes, values = module.call(g)
            assert np.array_equal(nodes, gids)  # rows come in dense order
            rows = rows_of(nodes, values)
            assert np.array_equal(rows, module_oracle(gids, src, dst))
            assert rows[:, 1].tolist() == expected  # networkx's partition, numbered canonically
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_analytical_and_transactional_mode():
    gids = np.array([30, 10, 20, 70, 50, 90, 80], dtype=np.int64)
    src, dst = np.array([10, 20, 30, 70, 50, 90]), np.array([20, 30, 10, 50, 70, 80])
    with Module(MODULE_SO) as module:
        with Graph(gids, src, dst) as g:
            assert np.array_equal(rows_of(*module.call(g)), module_oracle(gids, src, dst))
            g.hide_vertex(20)
            with pytest.raises(ProcedureError, match=r"^strongly_connected_components\.get: Invalid ID!$"):
                module.call(g)
        with Graph(gids, src, dst, transactional=False) as g:
            g.hide_vertex(80)  # a singleton: number 2 stays used, 90 is still 3
            rows = rows_of(*module.call(g))
            assert np.array_equal(rows, module_oracle(gids, src, dst, hidden=[80]))
            assert rows[:, 1].tolist() == [0, 0, 0, 1, 1, 3]

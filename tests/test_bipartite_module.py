"""bipartite_matching.so (memgraph_b200/csrc/bipartite_matching_module.cpp) on the in-memory mgp host with an
INTEGER-column call (tests/mgp_wcc_host.cpp; child interpreters as in tests/test_wcc_module.py).  No-GPU part: exports
and imports, the registered signature against the reference module's, one row with 0 for an empty graph and for a
graph without edges (no device touched).  GPU part (-m gpu): every graph of tests/golden/bipartite_cases.json gives the
reference's row, and the host's abort flag gives the procedure error."""
import os
import subprocess

import numpy as np
import pytest

import conftest
from _bc_host import REPO, isolated
from test_bc_module import PAGERANK_IMPORTS
from test_bipartite_oracle import REF_MODULE_SO, e2e_cases, golden, seeded_graphs, split, unit_cases
from test_wcc_module import Graph, Module, ProcedureError, host, live_objects

MODULE_SO = os.path.join(REPO, "memgraph_b200", "_build", "bipartite_matching.so")
SIGNATURE = "max() :: (maximum_bipartite_matching :: INTEGER)"


def call(module, n, f, t, gid_base=1000, abort=False):
    """One CALL on a graph of n vertices with gids gid_base + 3 * dense id -> the single row's value."""
    gids = gid_base + 3 * np.arange(n, dtype=np.int64)
    with Graph(gids, gids[np.asarray(f, dtype=np.int64)], gids[np.asarray(t, dtype=np.int64)]) as g:
        if abort:
            host().fh_graph_set_abort(g.h, 1)
        nodes, values = module.call(g, proc="max", column="maximum_bipartite_matching")
    assert len(values) == 1, len(values)
    return int(values[0])


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
def test_signature_is_the_reference_signature():
    with Module(MODULE_SO) as module:
        assert module.signature("max") == SIGNATURE
    if os.path.exists(REF_MODULE_SO):
        with Module(REF_MODULE_SO) as ref:
            assert ref.signature("max") == SIGNATURE


@isolated
def test_empty_graph_and_graph_without_edges():
    before = live_objects()
    with Module(MODULE_SO) as module:
        assert call(module, 0, [], []) == 0
        assert call(module, 5, [], []) == 0
        if not conftest.HAVE_GPU:
            with pytest.raises(ProcedureError, match=r"^bipartite_matching\.max: CUDA error"):
                call(module, 3, [0], [1])
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_rows_equal_the_reference_rows():
    before = live_objects()
    cases = [(name, n, *split(edges), expected) for name, n, edges, expected in list(e2e_cases()) + list(unit_cases())]
    cases += [(name, n, f, t, rec["expected"]) for (name, n, f, t), rec in zip(seeded_graphs(), golden()["seeded"])]
    with Module(MODULE_SO) as module:
        for name, n, f, t, expected in cases:
            assert call(module, n, f, t) == expected, name
    assert live_objects() == before


@pytest.mark.gpu
@isolated
def test_abort_flag_gives_the_error():
    before = live_objects()
    with Module(MODULE_SO) as module:
        with pytest.raises(ProcedureError, match=r"^bipartite_matching\.max: procedure aborted by the host$"):
            call(module, 4, [0, 1, 2], [1, 2, 3], abort=True)
        assert call(module, 4, [0, 1, 2], [1, 2, 3]) == 2  # the same module answers once the flag is down
    assert live_objects() == before

"""cugraph.pagerank.so / cugraph.personalized_pagerank.so (csrc/cugraph_modules.cpp): stand-ins for the reference's cuGraph
PageRank query modules, loaded through the fake mgp host.  No-GPU part: signatures identical to the reference modules'
registration (pagerank.cu:121-143, personalized_pagerank.cu:178-215), strict argument typing, no-device error text.
GPU part (-m gpu): the reference's e2e fixtures through the module, weights through the edge property, isolated vertices."""
import os

import numpy as np
import pytest

import _fakehost as fh
import conftest
from test_cugraph_oracle import FIXTURES, oracle_cugraph_pagerank

needs_modules = pytest.mark.skipif(not os.path.exists(fh.CUGRAPH_PAGERANK_SO), reason="modules not built")


@needs_modules
def test_signatures_match_the_reference_modules():
    with fh.Module(fh.CUGRAPH_PAGERANK_SO) as m:
        assert m.signature("get") == ("get(max_iterations = 100 :: INTEGER, damping_factor = 0.84999999999999998 :: FLOAT, "
                                      "stop_epsilon = 1.0000000000000001e-05 :: FLOAT, weight_property = \"weight\" :: STRING) :: "
                                      "(node :: NODE, pagerank :: FLOAT)")
    with fh.Module(fh.CUGRAPH_PERSONALIZED_SO) as m:
        assert m.signature("get") == ("get(personalization_vertices :: LIST OF NODE, personalization_values :: LIST OF FLOAT, "
                                      "max_iterations = 100 :: INTEGER, damping_factor = 0.84999999999999998 :: FLOAT, "
                                      "stop_epsilon = 1.0000000000000001e-05 :: FLOAT, weight_property = \"weight\" :: STRING) :: "
                                      "(node :: NODE, pagerank :: FLOAT)")


@needs_modules
def test_argument_errors_need_no_device():
    gids = [1, 2, 3]
    with fh.Module(fh.CUGRAPH_PERSONALIZED_SO) as m, fh.Graph(gids, [1, 2], [2, 3]) as g:
        with pytest.raises(fh.ProcedureError, match="requires between 2 and 6 arguments"):
            m.call(g)
        with pytest.raises(fh.ProcedureError, match="must have the same length"):
            m.call(g, [fh.Node(1)], [0.5, 0.5])
        nodes, ranks = m.call(g, [], [])  # no seeds: no rows, before any device work (:74)
        assert len(nodes) == 0
        with pytest.raises(fh.ProcedureError, match="must be of type INTEGER"):
            m.call(g, [fh.Node(1)], [1.0], 10.0)
    with fh.Module(fh.CUGRAPH_PAGERANK_SO) as m, fh.Graph([5, 6], [], []) as g:
        nodes, ranks = m.call(g)  # vertices but no edge: cuGraph knows no vertex, no rows, no device needed
        assert len(nodes) == 0
    assert fh.host().fh_live_objects() == 0


@needs_modules
@pytest.mark.skipif(conftest.HAVE_GPU, reason="this is the no-device behaviour")
def test_no_device_is_a_loud_procedure_error():
    with fh.Module(fh.CUGRAPH_PAGERANK_SO) as m, fh.Graph([1, 2], [1], [2]) as g:
        with pytest.raises(fh.ProcedureError, match="CUDA error"):
            m.call(g)


def _fixture_graph(fx):
    gids = fx["nodes"]
    return gids, [a for a, _ in fx["edges"]], [b for _, b in fx["edges"]]


@pytest.mark.gpu
@needs_modules
@pytest.mark.parametrize("fx", [f for f in FIXTURES if f["nodes"]], ids=lambda f: f["name"])
def test_reference_e2e_fixtures_through_the_modules(fx):
    gids, src, dst = _fixture_graph(fx)
    path = fh.CUGRAPH_PERSONALIZED_SO if fx["personalization"] else fh.CUGRAPH_PAGERANK_SO
    with fh.Module(path) as m, fh.Graph(gids, src, dst) as g:
        if fx["personalization"]:
            nodes, ranks = m.call(g, [fh.Node(v) for v, _ in fx["personalization"]], [x for _, x in fx["personalization"]])
        else:
            nodes, ranks = m.call(g)
    got = dict(zip(nodes.tolist(), ranks.tolist()))
    assert sorted(got) == sorted(gids)  # every fixture vertex has an edge: one row each
    for gid, want in fx["expected"]:
        digits = len(str(want).split(".")[1]) if "." in str(want) else 0
        assert abs(got[gid] - want) < max(1.5 * 10.0 ** -digits, 2e-5), (fx["name"], gid, got[gid], want)
    assert fh.host().fh_live_objects() == 0


@pytest.mark.gpu
@needs_modules
def test_weight_property_isolated_vertices_and_seeds():
    rng = np.random.default_rng(12)
    n, m = 400, 3000
    gids = (np.arange(n) * 7 + 100).tolist() + [99990, 99991]  # two isolated vertices at the end
    s, d = rng.integers(0, n, m), rng.integers(0, n, m)
    src, dst = [gids[i] for i in s], [gids[i] for i in d]
    w = rng.uniform(0.1, 4.0, m)
    w[:50] = np.nan  # edges without the property count 1.0
    used = sorted(set(src) | set(dst))
    dense = {g: i for i, g in enumerate(used)}
    f, t = [dense[x] for x in src], [dense[x] for x in dst]
    weights = np.where(np.isnan(w), 1.0, w)
    with fh.Module(fh.CUGRAPH_PAGERANK_SO) as m1, fh.Module(fh.CUGRAPH_PERSONALIZED_SO) as m2, fh.Graph(gids, src, dst) as g:
        g.set_edge_property("weight", src, w)
        nodes, ranks = m1.call(g, 100, 0.85, 1e-10)
        ref, _, _ = oracle_cugraph_pagerank(len(used), f, t, weights=weights, epsilon=1e-10)
        assert nodes.tolist() == used  # isolated vertices get no row
        assert float(np.max(np.abs(ranks - ref) / ref)) < 1e-9
        nodes2, ranks2 = m1.call(g, 100, 0.85, 1e-10, "no_such_property")  # every edge falls back to 1.0
        ref2, _, _ = oracle_cugraph_pagerank(len(used), f, t, epsilon=1e-10)
        assert float(np.max(np.abs(ranks2 - ref2) / ref2)) < 1e-9
        seeds = [fh.Node(used[3]), fh.Node(99990), fh.Node(used[17])]  # the isolated seed is skipped
        nodes3, ranks3 = m2.call(g, seeds, [0.2, 9.0, 0.5], 100, 0.85, 1e-10)
        ref3, _, _ = oracle_cugraph_pagerank(len(used), f, t, weights=weights, personalization=([3, 17], [0.2, 0.5]), epsilon=1e-10)
        assert float(np.max(np.abs(ranks3 - ref3) / np.maximum(ref3, 1e-3))) < 1e-9
        nodes4, _ = m2.call(g, [fh.Node(99991)], [1.0])  # only isolated seeds: no rows
        assert len(nodes4) == 0
        g.set_edge_property("weight", src, np.round(w), as_int=True)  # INTEGER-valued property is converted
        nodes5, ranks5 = m1.call(g, 100, 0.85, 1e-10)
        wi = np.where(np.isnan(w), 1.0, np.round(w))
        if (np.bincount(np.array(f), weights=wi, minlength=len(used)) >= 0).all():
            ref5, _, _ = oracle_cugraph_pagerank(len(used), f, t, weights=wi, epsilon=1e-10)
            assert float(np.max(np.abs(ranks5 - ref5) / ref5)) < 1e-9
    assert fh.host().fh_live_objects() == 0


@pytest.mark.gpu
@needs_modules
@pytest.mark.parametrize("env", [{"MGB200_IDX_FLAGS": "1"}, {"MGB200_FORCE_MULTI_PATH": "1"}])
def test_weight_property_under_gather_path_knobs(env, monkeypatch):
    """The gather-path knobs are tuning only: a weighted graph stays on the one gather path that has weights."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(13)
    n, m = 3000, 40000
    gids = (np.arange(n) * 3 + 11).tolist()
    s, d = rng.integers(0, n, m), rng.integers(0, n, m)
    src, dst = [gids[i] for i in s], [gids[i] for i in d]
    w = rng.uniform(0.1, 4.0, m)
    used = sorted(set(src) | set(dst))
    dense = {g: i for i, g in enumerate(used)}
    f, t = [dense[x] for x in src], [dense[x] for x in dst]
    with fh.Module(fh.CUGRAPH_PAGERANK_SO) as m1, fh.Graph(gids, src, dst) as g:
        g.set_edge_property("weight", src, w)
        nodes, ranks = m1.call(g, 100, 0.85, 1e-10)
    ref, _, _ = oracle_cugraph_pagerank(len(used), f, t, weights=w, epsilon=1e-10)
    assert nodes.tolist() == used
    assert float(np.max(np.abs(ranks - ref) / ref)) < 1e-9
    assert fh.host().fh_live_objects() == 0


@needs_modules
@pytest.mark.parametrize("path", [fh.CUGRAPH_PAGERANK_SO, fh.CUGRAPH_PERSONALIZED_SO, fh.BFS_MODULE_SO])
def test_modules_import_only_declared_mgp_symbols_and_no_cuda(path):
    """Loader contract (module.cpp:861 dlopen RTLD_NOW | RTLD_LOCAL): the module exports the two entry points, every undefined
    mgp_* symbol is one include/mgp_abi.h declares, and nothing CUDA / NCCL is left undefined (static runtime)."""
    import re
    import subprocess
    defined = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    assert " T mgp_init_module" in defined and " T mgp_shutdown_module" in defined
    und = subprocess.run(["nm", "-D", "--undefined-only", path], capture_output=True, text=True, check=True).stdout
    imported = {line.split()[-1] for line in und.splitlines() if " mgp_" in line}
    header = open(os.path.join(os.path.dirname(fh.REPO + "/"), "include", "mgp_abi.h")).read()
    declared = set(re.findall(r"\b(mgp_[a-z_0-9]+)\s*\(", header))
    assert imported <= declared, imported - declared
    assert "cuda" not in und.lower() and "nccl" not in und.lower()

"""-m gpu: the heavy rows' tile class (graph_build.cu tile_slices, pagerank_kernels.cu heavy_tiles_kernel).  A heavy row's
in-edges from the tiled hot prefix are summed per (row, tile) chunk from a shared-memory copy of that tile, the rest by
edge segments.  Only the order of the FP64 additions inside a heavy row may change: every layout the knobs allow must
match the oracle, repeat bit for bit, and count what scripts/tile_model.py counts."""
import os
import sys

import numpy as np
import pytest

from _checkers import Oracle

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
from tile_model import tile_model  # noqa: E402

REL_TOL = 1e-9


@pytest.fixture(scope="module")
def mg():
    import memgraph_b200
    return memgraph_b200


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def rel_err(got, ref):
    return float(np.max(np.abs(np.asarray(got) - ref) / ref))


def run_twice(mg, n, f, t, **kw):
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        info = dict(g.info)
        a, st = g.run(max_iterations=20, stop_epsilon=0.0, **kw)
        b, _ = g.run(max_iterations=20, stop_epsilon=0.0, **kw)
    assert st.iterations == 20
    assert np.array_equal(a, b)  # no float atomics: the same bits every run
    return a, info


def test_tiles_on_and_off_match_the_oracle(mg, oracle, monkeypatch):
    scale = 15
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m, seed=3)
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "64")
    on, info_on = run_twice(mg, n, f, t)
    monkeypatch.setenv("MGB200_TILE_LABELS", "0")
    off, info_off = run_twice(mg, n, f, t)
    ref, _ = oracle.pagerank(n, f, t, max_iterations=20, stop_epsilon=0.0)
    assert rel_err(on, ref) < REL_TOL and rel_err(off, ref) < REL_TOL
    assert rel_err(on, off) < 1e-12
    assert info_on["tiled_edges"] == info_on["heavy_edges"] > 0 and info_on["tile_chunks"] > 0  # 16 MB >= n labels
    assert info_off["tiled_edges"] == info_off["tile_chunks"] == 0
    assert info_on["heavy_segments"] == info_on["tile_chunks"]  # no cold edge left: every partial is a chunk


@pytest.mark.parametrize("scale,env", [
    (14, {"MGB200_TILE_LABELS": "2"}),                                   # smallest tile: one label pair per tile
    (14, {"MGB200_TILE_LABELS": "3000"}),                                # T does not divide H (= n here: H >= n)
    (14, {"MGB200_TILE_CHUNK": "1"}),                                    # one edge per chunk
    (14, {"MGB200_HEAVY_MIN_DEGREE": "2", "MGB200_TILE_CHUNK": "5"}),    # most rows heavy and tiled
    (14, {"MGB200_TILE_HOT_MB": "0"}),                                   # no tiles: every heavy edge cold
    (18, {"MGB200_TILE_HOT_MB": "1", "MGB200_TILE_LABELS": "10000"}),    # H = 2^17 < n: hot and cold edges per row
    (18, {"MGB200_TILE_HOT_MB": "1", "MGB200_HEAVY_MIN_DEGREE": "16", "MGB200_SEGMENT_EDGES": "64"}),
])
def test_tile_layouts_match_the_oracle_and_the_model(mg, oracle, monkeypatch, scale, env):
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m, seed=scale)
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "64")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    got, info = run_twice(mg, n, f, t)
    ref, _ = oracle.pagerank(n, f, t, max_iterations=20, stop_epsilon=0.0)
    assert rel_err(got, ref) < REL_TOL
    model = tile_model(n, f, t, tile_labels=int(os.environ.get("MGB200_TILE_LABELS", "16384")),
                       tile_hot_mb=int(os.environ.get("MGB200_TILE_HOT_MB", "16")),
                       tile_chunk=int(os.environ.get("MGB200_TILE_CHUNK", "256")),
                       heavy_min=int(os.environ["MGB200_HEAVY_MIN_DEGREE"]))
    assert (info["heavy_rows"], info["heavy_edges"]) == (model["heavy_rows"], model["heavy_edges"])
    assert (info["tiled_edges"], info["tile_chunks"]) == (model["tiled_edges"], model["tile_chunks"])
    assert info["heavy_segments"] >= info["tile_chunks"] + (info["heavy_edges"] > info["tiled_edges"])


def test_self_loops_multi_edges_and_cold_only_rows(mg, oracle, monkeypatch):
    """A hub fed by a few sources many times over (multi-edges, its own self-loop) next to a heavy row whose sources all
    lie past the tiled prefix."""
    rng = np.random.default_rng(17)
    n = 300_000
    hub_f = np.concatenate([rng.integers(0, 40, 5000), np.zeros(300, dtype=np.int64)])
    cold_f = rng.integers(200_000, n, 3000)
    # vertices >= 200000 receive no edge: in-degree 0 puts them past label 173 K, outside the 2^17-label tiled prefix
    f = np.concatenate([hub_f, cold_f, rng.integers(0, n, 400_000)])
    t = np.concatenate([np.zeros(len(hub_f), dtype=np.int64), np.full(len(cold_f), 1), rng.integers(0, 200_000, 400_000)])
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "64")
    monkeypatch.setenv("MGB200_TILE_HOT_MB", "1")
    monkeypatch.setenv("MGB200_TILE_LABELS", "4096")
    got, info = run_twice(mg, n, f, t)
    ref, _ = oracle.pagerank(n, f, t, max_iterations=20, stop_epsilon=0.0)
    assert rel_err(got, ref) < REL_TOL
    assert 0 < info["tiled_edges"] < info["heavy_edges"]
    model = tile_model(n, f, t, tile_labels=4096, tile_hot_mb=1, heavy_min=64)
    assert (info["tiled_edges"], info["tile_chunks"]) == (model["tiled_edges"], model["tile_chunks"])


def test_katz_bit_exact_with_small_tiles(monkeypatch):
    import memgraph_b200 as mg
    from test_gpu_katz import check
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "16")
    monkeypatch.setenv("MGB200_TILE_LABELS", "64")
    monkeypatch.setenv("MGB200_TILE_CHUNK", "7")
    scale = 12
    n, m = 1 << scale, 8 << scale
    f, t = mg.rmat_edges_host(scale, m, seed=9)
    deg_max = np.bincount(f.astype(np.int64), minlength=n).max()
    st = check(n, f, t, alpha=float(0.9 / np.sqrt(deg_max + 1.0)), eps=1e-3)
    assert st["iterations"] >= 2


def test_personalised_pagerank_reproducible_with_tiles(monkeypatch):
    import memgraph_b200 as mg
    from memgraph_b200 import personalized as P
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "32")
    monkeypatch.setenv("MGB200_TILE_LABELS", "512")
    scale = 16
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    seeds = (np.array([0, 1234, 40000]), np.array([0.2, 0.5, 0.3]))
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        assert g.info["tiled_edges"] > 0
        a, _ = P.cugraph_pagerank(g, *seeds, max_iterations=20, stop_epsilon=0.0)
        b, _ = P.cugraph_pagerank(g, *seeds, max_iterations=20, stop_epsilon=0.0)
    monkeypatch.setenv("MGB200_TILE_LABELS", "0")
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        off, _ = P.cugraph_pagerank(g, *seeds, max_iterations=20, stop_epsilon=0.0)
    assert np.array_equal(a, b)
    assert float(np.max(np.abs(a - off))) < 1e-12 * float(np.max(off))  # vertices no seed reaches stay exactly 0


def test_lone_partition_builds_per_owner_tiles(mg, monkeypatch):
    """Partition 1 of 4 on one GPU (no peers): its heavy rows' sources fall in all four owners' hot prefixes, each cut
    into its own tiles (the owners' first labels are odd here, so tiles start one label early).  The ranks are not
    PageRank's (no peer pushes), but the same inputs must give the same numbers with tiles on and off."""
    scale = 16
    n, m = (1 << scale) + 3, 16 << scale
    f, t = mg.rmat_edges_host(scale, m, seed=5)
    monkeypatch.setenv("MGB200_LONE_PARTITION", "1")
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "32")
    monkeypatch.setenv("MGB200_TILE_LABELS", "1000")
    out = {}
    for tiles in ("1000", "0"):
        monkeypatch.setenv("MGB200_TILE_LABELS", tiles)
        with mg.PageRankGraph.from_arrays(n, f, t, part_rank=1, part_world=4) as g:
            info = dict(g.info)
            a, va, _ = g.run_partition(max_iterations=10, stop_epsilon=0.0)
            b, _, _ = g.run_partition(max_iterations=10, stop_epsilon=0.0)
        assert np.array_equal(a, b)
        out[tiles] = (a, va, info)
    (on, v_on, i_on), (off, v_off, i_off) = out["1000"], out["0"]
    assert i_on["tiled_edges"] == i_on["heavy_edges"] > 0 and i_off["tiled_edges"] == 0
    assert np.array_equal(v_on, v_off)
    assert float(np.max(np.abs(on - off) / off)) < 1e-12

"""-m gpu: the block class (graph_build.cu block_edges and block_slices, pagerank_kernels.cu cold_block_kernel).  The
heavy rows' in-edges from labels >= MGB200_BLOCK_FROM are summed one label block at a time into partials of their
own.  Only the order of the FP64 additions inside a heavy row may change: every layout the knobs allow must match the
oracle, repeat bit for bit, agree with the class turned off, and count what scripts/block_model.py counts."""
import os
import sys

import numpy as np
import pytest

from _checkers import Oracle

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
from block_model import block_model  # noqa: E402

REL_TOL = 1e-9
ZERO, SELL, SELL_EPI, HEAVY_SEG, HEAVY_FIN, ITER_END = range(6)  # core.hpp Graph::kCls*


@pytest.fixture(scope="module")
def mg():
    import memgraph_b200
    return memgraph_b200


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def rel_err(got, ref):
    return float(np.max(np.abs(np.asarray(got) - ref) / ref))


def run_twice(mg, n, f, t, iters=20):
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        info = dict(g.info)
        a, st = g.run(max_iterations=iters, stop_epsilon=0.0)
        b, _ = g.run(max_iterations=iters, stop_epsilon=0.0)
    assert st.iterations == iters
    assert np.array_equal(a, b)  # no float atomics: the same bits every run
    return a, info


def model_for(n, f, t):
    e = os.environ
    return block_model(n, f, t, block_from=int(e.get("MGB200_BLOCK_FROM", 2 << 20)),
                       block_labels=int(e.get("MGB200_BLOCK_LABELS", 2 << 20)),
                       block_chunk=int(e.get("MGB200_BLOCK_CHUNK", 16)),
                       heavy_min=int(e.get("MGB200_HEAVY_MIN_DEGREE", 1024)))


def check_against_model(info, model):
    keys = ("heavy_rows", "heavy_edges", "block_edges", "block_chunks", "blocks")
    assert tuple(info[k] for k in keys) == tuple(model[k] for k in keys)


LAYOUTS = {  # scale, environment
    "blocks_divide_n": (16, {"MGB200_BLOCK_FROM": "4096", "MGB200_BLOCK_LABELS": "4096"}),
    "blocks_do_not_divide_n": (16, {"MGB200_BLOCK_FROM": "1000", "MGB200_BLOCK_LABELS": "7777"}),
    "one_label_per_block": (12, {"MGB200_BLOCK_FROM": "3000", "MGB200_BLOCK_LABELS": "1"}),
    "chunk_cap_1": (15, {"MGB200_BLOCK_FROM": "2000", "MGB200_BLOCK_LABELS": "5000", "MGB200_BLOCK_CHUNK": "1"}),
    "from_below_tiles": (16, {"MGB200_BLOCK_FROM": "20000", "MGB200_BLOCK_LABELS": "9000", "MGB200_TILE_HOT_MB": "1"}),
    "from_equal_tiles": (18, {"MGB200_BLOCK_FROM": "131072", "MGB200_BLOCK_LABELS": "30000", "MGB200_TILE_HOT_MB": "1"}),
    "from_above_tiles": (18, {"MGB200_BLOCK_FROM": "140000", "MGB200_BLOCK_LABELS": "20000", "MGB200_TILE_HOT_MB": "1",
                              "MGB200_SEGMENT_EDGES": "64"}),
    "from_zero": (14, {"MGB200_BLOCK_FROM": "0", "MGB200_BLOCK_LABELS": "3000"}),
    "tiles_off": (16, {"MGB200_BLOCK_FROM": "3000", "MGB200_BLOCK_LABELS": "10000", "MGB200_TILE_LABELS": "0"}),
    "block_count_capped": (14, {"MGB200_BLOCK_FROM": "0", "MGB200_BLOCK_LABELS": "1"}),  # 16 K labels, <= 4096 blocks
}


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_block_layouts_match_the_oracle_the_model_and_the_class_off(mg, oracle, monkeypatch, name):
    scale, env = LAYOUTS[name]
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m, seed=scale + 1)
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "64")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    on, info = run_twice(mg, n, f, t)
    ref, _ = oracle.pagerank(n, f, t, max_iterations=20, stop_epsilon=0.0)
    assert rel_err(on, ref) < REL_TOL
    assert info["block_edges"] > 0 and info["blocks"] > 0
    check_against_model(info, model_for(n, f, t))
    monkeypatch.setenv("MGB200_BLOCK_LABELS", "0")
    off, info_off = run_twice(mg, n, f, t)
    assert info_off["block_edges"] == info_off["block_chunks"] == info_off["blocks"] == 0
    assert info["sell_entries"] == info_off["sell_entries"]  # the SELL rows keep every column
    assert info["blocks"] <= 4096
    assert rel_err(on, off) < 1e-13


def test_cold_only_heavy_row_self_loops_and_multi_edges(mg, oracle, monkeypatch):
    """A heavy row whose every source lies past the bound (no tile chunk, no segment: block chunks only), next to a hub fed
    by a few sources many times over (multi-edges, its own self-loop) and heavy rows with both kinds of source."""
    rng = np.random.default_rng(23)
    n = 200_000
    hub_f = np.concatenate([rng.integers(0, 40, 4000), np.zeros(200, dtype=np.int64)])
    far = np.arange(100_000, n)  # in-degree 0: labelled past every vertex with in-edges
    cold_hub_f = rng.choice(far, 3000)
    f = np.concatenate([hub_f, cold_hub_f, rng.integers(0, n, 300_000)])
    t = np.concatenate([np.zeros(len(hub_f), dtype=np.int64), np.full(len(cold_hub_f), 1), rng.integers(2, 100_000, 300_000)])
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "16")
    monkeypatch.setenv("MGB200_TILE_HOT_MB", "0")  # the sources below the bound go to segments
    monkeypatch.setenv("MGB200_BLOCK_FROM", "60000")
    monkeypatch.setenv("MGB200_BLOCK_LABELS", "15000")
    got, info = run_twice(mg, n, f, t)
    ref, _ = oracle.pagerank(n, f, t, max_iterations=20, stop_epsilon=0.0)
    assert rel_err(got, ref) < REL_TOL
    check_against_model(info, model_for(n, f, t))
    assert info["tiled_edges"] == 0 < info["block_edges"] < info["heavy_edges"]  # the hub's edges below the bound: segments


def test_katz_bit_exact_with_the_class_on_and_off(monkeypatch):
    import memgraph_b200 as mg
    from memgraph_b200 import katz
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "16")
    monkeypatch.setenv("MGB200_BLOCK_FROM", "500")
    monkeypatch.setenv("MGB200_BLOCK_CHUNK", "7")
    scale = 13
    n, m = 1 << scale, 8 << scale
    f, t = mg.rmat_edges_host(scale, m, seed=9)
    alpha = float(0.9 / np.sqrt(np.bincount(f.astype(np.int64), minlength=n).max() + 1.0))
    out = {}
    for labels in ("999", "0"):
        monkeypatch.setenv("MGB200_BLOCK_LABELS", labels)
        with mg.PageRankGraph.from_arrays(n, f, t) as g:
            assert (g.info["blocks"] > 0) == (labels != "0")
            out[labels], st = katz.set_katz(g, alpha=alpha, epsilon=1e-3)
        assert st["iterations"] >= 2
    assert np.array_equal(out["999"], out["0"])


@pytest.mark.parametrize("seeds", [None, (np.array([0, 1234, 4000]), np.array([0.2, 0.5, 0.3]))],
                         ids=["uniform", "seeded"])
def test_personalised_pagerank_with_blocks(monkeypatch, seeds):
    import memgraph_b200 as mg
    from memgraph_b200 import personalized as P
    from test_cugraph_oracle import oracle_cugraph_pagerank
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "32")
    monkeypatch.setenv("MGB200_BLOCK_FROM", "1500")
    scale = 13
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    out = {}
    for labels in ("5000", "0"):
        monkeypatch.setenv("MGB200_BLOCK_LABELS", labels)
        with mg.PageRankGraph.from_arrays(n, f, t) as g:
            assert (g.info["blocks"] > 0) == (labels != "0")
            a, _ = P.cugraph_pagerank(g, *(seeds or ()), max_iterations=20, stop_epsilon=0.0)
            b, _ = P.cugraph_pagerank(g, *(seeds or ()), max_iterations=20, stop_epsilon=0.0)
        assert np.array_equal(a, b)
        out[labels] = a
    assert float(np.max(np.abs(out["5000"] - out["0"]))) < 1e-12 * float(np.max(out["0"]))
    ref, _, _ = oracle_cugraph_pagerank(n, f, t, personalization=seeds, alpha=0.85, epsilon=0.0, max_iterations=20)
    assert float(np.max(np.abs(out["5000"] - ref))) < REL_TOL * float(np.max(ref))


def test_weighted_and_lone_partition_builds_have_no_blocks(mg, monkeypatch):
    from memgraph_b200 import personalized as P
    monkeypatch.setenv("MGB200_BLOCK_FROM", "100")
    monkeypatch.setenv("MGB200_BLOCK_LABELS", "1000")
    rng = np.random.default_rng(6)
    n = 4000
    f, t = rng.integers(0, n, 40_000), rng.integers(0, n, 40_000)
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "8")
    with P.weighted_graph(n, f, t, rng.uniform(0.5, 2.0, len(f))) as g:
        assert g.info["block_edges"] == g.info["blocks"] == 0
    monkeypatch.setenv("MGB200_LONE_PARTITION", "1")
    with mg.PageRankGraph.from_arrays(n, f, t, part_rank=1, part_world=2) as g:
        assert g.info["block_edges"] == g.info["blocks"] == 0
    monkeypatch.delenv("MGB200_LONE_PARTITION")
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        assert g.info["block_edges"] > 0 and g.info["blocks"] == 4


LAUNCH_CONFIGS = {  # environment; the tiled prefix (16 MB) reaches past the bound, so no heavy row has CSC segments
    "blocks_heavy_and_sell": {"MGB200_HEAVY_MIN_DEGREE": "64", "MGB200_BLOCK_FROM": "4096", "MGB200_BLOCK_LABELS": "6000"},
    "blocks_no_sell_rows": {"MGB200_HEAVY_MIN_DEGREE": "2", "MGB200_BLOCK_FROM": "1000", "MGB200_BLOCK_LABELS": "700"},
}


def launch_graph(name):
    import memgraph_b200 as mg
    if name == "blocks_no_sell_rows":  # every edge twice: each in-degree is 0 or >= 2
        rng = np.random.default_rng(4)
        f, t = rng.integers(0, 3000, 20_000), rng.integers(0, 3000, 20_000)
        return 3000, np.concatenate([f, f]), np.concatenate([t, t])
    return (1 << 15, *mg.rmat_edges_host(15, 16 << 15, seed=15))


@pytest.fixture(params=sorted(LAUNCH_CONFIGS))
def launch_config(request, monkeypatch):
    for k, v in LAUNCH_CONFIGS[request.param].items():
        monkeypatch.setenv(k, v)
    return request.param, launch_graph(request.param)


def gather_launches(info, row_sums):
    sell, heavy, tiles = info["sell_slices"] > 0, info["heavy_segments"] > 0, info["tile_chunks"] > 0
    return sell + info["blocks"] + tiles + (heavy and row_sums)  # no CSC segments: every cold edge is in a block


def test_launch_counts_with_blocks(launch_config):
    import memgraph_b200 as mg
    from memgraph_b200 import katz
    from memgraph_b200 import personalized as P
    name, (n, f, t) = launch_config
    k = 3
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        info = dict(g.info)
        _, st = g.run(max_iterations=k, stop_epsilon=0.0, time_spmv_kernel=True)
        deg_max = int(np.bincount(np.asarray(f, dtype=np.int64), minlength=n).max())
        _, kst = katz.set_katz(g, alpha=0.9 / float(np.sqrt(deg_max + 1.0)), epsilon=1e-3)
        _, pst = P.cugraph_pagerank(g, max_iterations=6, stop_epsilon=0.0)
    sell, heavy = info["sell_slices"] > 0, info["heavy_segments"] > 0
    assert info["blocks"] > 0 and heavy and sell == (name == "blocks_heavy_and_sell")
    tiles = info["tile_chunks"] > 0
    assert tiles and info["tiled_edges"] + info["block_edges"] >= info["heavy_edges"] > 0
    zero_refresh = info["zero_rows"] > 0
    assert st.kernel_launches == k * (1 + 2 * sell + info["blocks"] + heavy * (2 + tiles)) + zero_refresh + 2
    assert st.class_ms[SELL] > 0.0 if sell else st.class_ms[SELL] == 0.0
    it = kst["iterations"]
    per_iteration = gather_launches(info, row_sums=False) + (info["sell_rows"] > 0) + (info["heavy_rows"] > 0) + 6
    zero_fill = it >= 2 and info["zero_rows"] > 0
    assert kst["kernel_launches"] == 2 + it * per_iteration + zero_fill + 3 * kst["tie_order_runs"] + 1
    assert pst["kernel_launches"] == 1 + 6 * (4 + gather_launches(info, row_sums=True)) + 1

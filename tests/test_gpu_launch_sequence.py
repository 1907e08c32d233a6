"""-m gpu: the kernel sequence of the gather paths.  PageRank, Katz and personalised PageRank launch the same gather (SELL
row sums, then heavy-row partials from the tiles and the cold segments); which of its kernels run depends only on the
row classes the build made, so every entry point's `kernel_launches` is a closed formula of the graph's info fields.
With per-kernel timing on, PageRank's `class_ms` must be zero for every kernel class it did not launch and positive for
the ones it did."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ZERO, SELL, SELL_EPI, HEAVY_SEG, HEAVY_FIN, ITER_END = range(6)  # core.hpp Graph::kCls*


def rmat(scale):
    import memgraph_b200 as mg
    n, m = 1 << scale, 16 << scale
    return (n, *mg.rmat_edges_host(scale, m, seed=scale))


def uniform(n=10_000, m=50_000, seed=3):
    rng = np.random.default_rng(seed)
    return n, rng.integers(0, n, m), rng.integers(0, n, m)


def doubled(n=3000, m=20_000, seed=4):
    """Every edge twice: each in-degree is 0 or >= 2, so MGB200_HEAVY_MIN_DEGREE=2 leaves no SELL row."""
    n, f, t = uniform(n, m, seed)
    return n, np.concatenate([f, f]), np.concatenate([t, t])


# (graph, environment, PageRank iterations)
CONFIGS = {
    "all_heavy_edges_tiled": (lambda: rmat(14), {"MGB200_HEAVY_MIN_DEGREE": "64"}, 5),
    "all_heavy_edges_cold": (lambda: rmat(14), {"MGB200_HEAVY_MIN_DEGREE": "64", "MGB200_TILE_LABELS": "0"}, 5),
    "tiled_and_cold_edges": (lambda: rmat(18), {"MGB200_HEAVY_MIN_DEGREE": "64", "MGB200_TILE_HOT_MB": "1"}, 4),
    "no_overlap_epilogue": (lambda: rmat(18), {"MGB200_HEAVY_MIN_DEGREE": "64", "MGB200_TILE_HOT_MB": "1",
                                               "MGB200_OVERLAP_EPILOGUE": "0"}, 3),
    "no_heavy_rows": (uniform, {}, 1),
    "no_sell_rows": (doubled, {"MGB200_HEAVY_MIN_DEGREE": "2"}, 2),
}


@pytest.fixture(params=sorted(CONFIGS))
def config(request, monkeypatch):
    make, env, iters = CONFIGS[request.param]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return request.param, make(), iters


def classes(info):
    """Which parts of the gather this graph has: SELL slices, heavy rows, tile chunks, cold segments."""
    heavy = info["heavy_segments"] > 0
    return (info["sell_slices"] > 0, heavy, heavy and info["tile_chunks"] > 0,
            heavy and info["heavy_segments"] > info["tile_chunks"])


def gather_launches(info, row_sums):
    sell, heavy, tiles, cold = classes(info)
    return sell + tiles + cold + (heavy and row_sums)


def check_layout(name, info):
    sell, heavy, tiles, cold = classes(info)
    expect = {"all_heavy_edges_tiled": (True, True, True, False), "all_heavy_edges_cold": (True, True, False, True),
              "tiled_and_cold_edges": (True, True, True, True), "no_overlap_epilogue": (True, True, True, True),
              "no_heavy_rows": (True, False, False, False), "no_sell_rows": (False, True, True, False)}[name]
    assert (sell, heavy, tiles, cold) == expect, (name, info)


def test_pagerank_launch_count_and_class_timing(config):
    import memgraph_b200 as mg
    name, (n, f, t), k = config
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        info = dict(g.info)
        _, st = g.run(max_iterations=k, stop_epsilon=0.0, time_spmv_kernel=True)
    check_layout(name, info)
    sell, heavy, tiles, cold = classes(info)
    zero_refresh = k >= 2 and info["zero_rows"] > 0
    assert st.iterations == k
    assert st.kernel_launches == k * (1 + 2 * sell + heavy * (2 + tiles + cold)) + zero_refresh + 2
    assert st.spmv_launches == k * sell
    launched = {ZERO: zero_refresh, SELL: sell, SELL_EPI: sell, HEAVY_SEG: heavy, HEAVY_FIN: heavy, ITER_END: True}
    for cls, on in launched.items():
        if not on:
            assert st.class_ms[cls] == 0.0, (cls, st.class_ms)
        elif cls != ZERO:  # one short refresh kernel may fall below the events' resolution
            assert st.class_ms[cls] > 0.0, (cls, st.class_ms)
    assert st.kernel_ms == st.class_ms[SELL]


def test_katz_launch_count(config):
    import memgraph_b200 as mg
    from memgraph_b200 import katz
    name, (n, f, t), _ = config
    deg_max = int(np.bincount(np.asarray(f, dtype=np.int64), minlength=n).max())
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        info = dict(g.info)
        _, st = katz.set_katz(g, alpha=0.9 / float(np.sqrt(deg_max + 1.0)), epsilon=1e-3)
    check_layout(name, info)
    it = st["iterations"]
    per_iteration = gather_launches(info, row_sums=False) + (info["sell_rows"] > 0) + (info["heavy_rows"] > 0) + 6
    zero_fill = it >= 2 and info["zero_rows"] > 0
    assert it >= 1
    assert st["kernel_launches"] == 2 + it * per_iteration + zero_fill + 3 * st["tie_order_runs"] + 1


@pytest.mark.parametrize("seeds", [None, (np.array([0, 17, 400]), np.array([0.2, 0.5, 0.3]))], ids=["uniform", "seeded"])
def test_personalized_pagerank_launch_count(config, seeds):
    import memgraph_b200 as mg
    from memgraph_b200 import personalized as P
    name, (n, f, t), _ = config
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        info = dict(g.info)
        _, st = P.cugraph_pagerank(g, *(seeds or ()), max_iterations=6, stop_epsilon=0.0)
    check_layout(name, info)
    assert st["iterations"] == 6
    assert st["kernel_launches"] == 1 + 6 * (4 + gather_launches(info, row_sums=True)) + 1


@pytest.mark.parametrize("heavy_min", ["16", "1024"])
def test_personalized_pagerank_launch_count_weighted(monkeypatch, heavy_min):
    """The weighted handle gathers through the weighted SELL and heavy-segment kernels and has no tile class."""
    from memgraph_b200 import personalized as P
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", heavy_min)
    n, f, t = uniform(4000, 40_000, seed=5)
    w = np.random.default_rng(6).uniform(0.5, 2.0, len(f))
    with P.weighted_graph(n, f, t, w) as g:
        info = dict(g.info)
        _, st = P.cugraph_pagerank(g, max_iterations=6, stop_epsilon=0.0)
    sell, heavy, tiles, cold = classes(info)
    assert sell and heavy == (heavy_min == "16") and not tiles and cold == heavy
    assert st["iterations"] == 6
    assert st["kernel_launches"] == 1 + 6 * (4 + gather_launches(info, row_sums=True)) + 1

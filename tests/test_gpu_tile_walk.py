"""-m gpu: how heavy_tiles_kernel walks the tile slices (pagerank_kernels.cu tile_walk).  Persistent CTAs draw runs of
slices from a ticket in tile order; inside a run the warps draw groups of consecutive slices and walk each group as one
stream of columns, a slice boundary only deciding where a lane's sum is stored.  None of that may change a bit of any
partial, so every shape of run, group and slice below must match the oracle, agree with the tiles turned off, and
repeat byte for byte -- also on a handle that has run before, whether that run went to its last iteration or not.
With the default 8 runs per SM a group of more than one slice needs millions of chunks; MGB200_TILE_RUNS (the number
of runs) brings groups of up to 31 slices to graphs of 16 K vertices, and `info` (tile_slices, tile_runs) shows that a
case reached the group it is about.  The hub-graph cases have a handful of slices per run: groups of one slice."""
import numpy as np
import pytest

from _checkers import Oracle

pytestmark = pytest.mark.gpu

REL_TOL = 1e-9
UNROLL = 16  # kTileUnroll: columns per batch of the walk


@pytest.fixture(scope="module")
def mg():
    import memgraph_b200
    return memgraph_b200


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def rel_err(got, ref):
    return float(np.max(np.abs(np.asarray(got) - ref) / ref))


def hub_graph(n, hubs, seed, spread=None):
    """`hubs` = in-degrees of vertices 0..len(hubs)-1, each fed by distinct sources drawn from [len(hubs), spread); every
    other vertex gets one in-edge from its predecessor, so that only the hubs are heavy rows."""
    rng = np.random.default_rng(seed)
    h = len(hubs)
    spread = n if spread is None else spread
    f, t = [np.arange(h, n - 1, dtype=np.int64)], [np.arange(h + 1, n, dtype=np.int64)]
    for v, d in enumerate(hubs):
        f.append(rng.choice(np.arange(h, spread, dtype=np.int64), size=d, replace=False))
        t.append(np.full(d, v, dtype=np.int64))
    return np.concatenate(f), np.concatenate(t)


def check(mg, oracle, monkeypatch, n, f, t, env, expect_chunks=None):
    """Tiles on: oracle, twice the same bytes on one handle; tiles off: the same ranks to 1e-14."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        info = dict(g.info)
        a, st = g.run(max_iterations=20, stop_epsilon=0.0)
        b, _ = g.run(max_iterations=20, stop_epsilon=0.0)  # the run ticket was rewound by the first run's last launch
    assert st.iterations >= 2  # (a hub graph can reach a delta of exactly 0 before the 20th iteration)
    assert np.array_equal(a, b)
    assert info["tiled_edges"] > 0
    if expect_chunks is not None:
        assert info["tile_chunks"] == expect_chunks
    ref, _ = oracle.pagerank(n, f, t, max_iterations=20, stop_epsilon=0.0)
    assert rel_err(a, ref) < REL_TOL
    monkeypatch.setenv("MGB200_TILE_LABELS", "0")
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        assert g.info["tiled_edges"] == 0
        off, _ = g.run(max_iterations=20, stop_epsilon=0.0)
    assert rel_err(a, off) < 1e-14
    return info


def test_one_heavy_row_in_one_tile(mg, oracle, monkeypatch):
    """One chunk: a single slice with one live lane, one run, one group -- fewer slices than warps, CTAs or a group."""
    n = 4000
    f, t = hub_graph(n, [200], seed=1)
    check(mg, oracle, monkeypatch, n, f, t, {"MGB200_HEAVY_MIN_DEGREE": "64"}, expect_chunks=1)


def test_a_few_slices_in_one_tile(mg, oracle, monkeypatch):
    """70 chunks of different lengths in one tile: three slices (the last one with padding lanes), each its own run."""
    n = 6000
    f, t = hub_graph(n, [70 + 2 * i for i in range(70)], seed=2)
    check(mg, oracle, monkeypatch, n, f, t, {"MGB200_HEAVY_MIN_DEGREE": "64"}, expect_chunks=70)


@pytest.mark.parametrize("width", [1, UNROLL - 1, UNROLL, UNROLL + 1, 2 * UNROLL, 2 * UNROLL + 1])
def test_slice_width_against_the_batch(mg, oracle, monkeypatch, width):
    """Chunks capped at `width` edges: most slices are exactly that wide (one column, a batch less one, a full batch, a
    batch and one column, ...), the slices of the rows' last chunks are narrower."""
    n = 5000
    f, t = hub_graph(n, [40 * width + 3 * i for i in range(48)], seed=3 + width)
    check(mg, oracle, monkeypatch, n, f, t, {"MGB200_HEAVY_MIN_DEGREE": "32", "MGB200_TILE_CHUNK": str(width)})


def test_sources_spread_over_many_small_tiles(mg, oracle, monkeypatch):
    """64-label tiles: each hub's sources fall into ~60 tiles, a few chunks per tile, so most tiles hold one or two
    slices and every run ends where its tile does."""
    n = 4096
    f, t = hub_graph(n, [300 + 5 * i for i in range(40)], seed=11)
    info = check(mg, oracle, monkeypatch, n, f, t, {"MGB200_HEAVY_MIN_DEGREE": "64", "MGB200_TILE_LABELS": "64"})
    assert info["tile_chunks"] > 40 * 30


def largest_group(info, tiles):
    """A lower bound of the largest group of slices one warp ticket hands out.  The kernel cuts a run where it crosses
    into the next tile, so `tile_runs` runs over `tiles` tiles are walked in at most runs + tiles - 1 parts and one part
    holds at least the average; in a part of p slices a group is clamp(p / (16 warps * 4 groups per warp), 1, 31)."""
    parts = info["tile_runs"] + tiles - 1
    return min(31, max(1, -(-info["tile_slices"] // parts) // (16 * 4)))


@pytest.mark.parametrize("scale,chunk,runs,min_group", [
    (14, "3", "4", 8),    # one tile; slices 1-3 columns wide: many slices close inside one batch
    (14, "8", "2", 8),    # slices up to half a batch wide
    (14, "20", "1", 8),   # ONE run, so one CTA walks everything; boundaries inside and at the end of 16-column batches
    (14, "40", "1", 4),   # slices of up to two and a half batches: a whole batch, then a boundary in the middle of one
    (16, "12", "3", 8),   # four tiles, three runs: every run crosses a tile boundary and is walked in parts
    (16, "5", "8", 8),    # more runs than tiles
    (15, "2", "1", 31),   # two tiles of > 4000 narrow slices: the largest group, every lane holds a column base
])
def test_groups_of_several_slices(mg, oracle, monkeypatch, scale, chunk, runs, min_group):
    """Nearly every row heavy, chunks capped well below the default and only a few runs (MGB200_TILE_RUNS), so a part of
    a run holds hundreds of slices on a small graph and a warp's ticket covers a group of them: the group is one stream
    of columns in which slices of different widths close, its last slices are cut at the end of the part, and the
    offsets of the next slice are already requested when a slice closes."""
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m, seed=scale)
    info = check(mg, oracle, monkeypatch, n, f, t, {"MGB200_HEAVY_MIN_DEGREE": "2", "MGB200_TILE_CHUNK": chunk,
                                                   "MGB200_TILE_RUNS": runs})
    assert info["tile_runs"] == int(runs) and info["tile_slices"] * 32 >= info["tile_chunks"]
    assert largest_group(info, tiles=-(-n // 16384)) >= min_group
    if int(chunk) > 2:  # the slices are not all one column wide
        assert info["tiled_edges"] > 2 * info["tile_chunks"]


def test_wide_and_narrow_slices_with_cold_edges(mg, oracle, monkeypatch):
    """A 1 MB tiled prefix on a graph larger than it: wide slices in the first tiles, narrow ones in the last, and the
    rows' cold edges on the segment stream next to the tile kernel."""
    scale = 18
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m, seed=7)
    info = check(mg, oracle, monkeypatch, n, f, t, {"MGB200_HEAVY_MIN_DEGREE": "16", "MGB200_TILE_HOT_MB": "1",
                                                   "MGB200_TILE_LABELS": "4096"})
    assert 0 < info["tiled_edges"] < info["heavy_edges"]


def test_run_after_an_early_stop(mg, oracle, monkeypatch):
    """A run that converges before max_iterations leaves launches behind that return at once; the next run on the handle
    must find the run ticket at zero and give the bytes of a fresh handle."""
    scale = 16
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m, seed=21)
    env = {"MGB200_HEAVY_MIN_DEGREE": "32", "MGB200_TILE_CHUNK": "5", "MGB200_TILE_LABELS": "1024"}
    check(mg, oracle, monkeypatch, n, f, t, env)  # oracle, tiles off, two full runs on one handle
    monkeypatch.setenv("MGB200_TILE_LABELS", "1024")
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        assert g.info["tiled_edges"] > 0
        fresh, st = g.run(max_iterations=20, stop_epsilon=0.0)
        assert st.iterations == 20
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        early, st = g.run(max_iterations=100, stop_epsilon=1e-6)
        assert 1 < st.iterations < 100
        early2, st2 = g.run(max_iterations=100, stop_epsilon=1e-6)
        after, _ = g.run(max_iterations=20, stop_epsilon=0.0)
    assert st2.iterations == st.iterations and np.array_equal(early, early2)
    assert np.array_equal(after, fresh)
    ref, _ = oracle.pagerank(n, f, t, max_iterations=100, stop_epsilon=1e-6)
    assert rel_err(early, ref) < REL_TOL

"""The PageRank layout's gather (launch_gather_phase, through mgb200_graph_gather) as an exact SpMV.

PageRank, Katz, the cuGraph PageRanks and both HITS handles iterate one gather, y = A^T x.  When every x[v] is an integer
and every partial sum of a row stays below 2^53, y is exact in FP64 in any add order, so the gather must equal an exact
host reference bit for bit in every row, under every layout and gather variant.  One dropped, doubled or misrouted edge
moves some row by at least 2^(bits-1); a value stored or summed in FP32 anywhere on the path loses the low bits of
values drawn above 2^24.  The whole-algorithm comparisons elsewhere cannot see either: their vectors are positive,
smooth and dominated by a few hot sources, and one cold source's share of a row lies far below their 1e-9 tolerance.

Row classes and labels come from a host model of the build (graph_build.cu `labels`: in-degree descending, out-degree
descending, id ascending), so a failure names the first bad row, its label and its class.  Without a GPU, the file
checks that model against scripts/block_model.py and checks that every seam graph puts its rows and sources where the
GPU tests say they are."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
from block_model import block_model  # noqa: E402
from test_gpu_gather_variants import LAYOUT, VARIANTS, dyadic_weights, katz_alpha  # noqa: E402

gpu = pytest.mark.gpu
U = 2.0 ** -53  # unit roundoff of FP64

# ---- host model of the layout ----------------------------------------------------------------------------------------


class Model:
    """Labels and row classes of a single-partition build of (n, f, t) with heavy rows from in-degree `heavy_min`."""

    def __init__(self, n, f, t, heavy_min=1024):
        self.n = n
        self.f = np.asarray(f, dtype=np.int64)
        self.t = np.asarray(t, dtype=np.int64)
        self.indeg = np.bincount(self.t, minlength=n)
        self.outdeg = np.bincount(self.f, minlength=n)
        order = np.lexsort((np.arange(n), -self.outdeg, -self.indeg))  # label -> vertex
        self.vertex = order
        self.label = np.empty(n, dtype=np.int64)
        self.label[order] = np.arange(n)
        self.heavy_min = heavy_min
        self.n_heavy = int(np.count_nonzero(self.indeg >= heavy_min))
        self.n_sell = int(np.count_nonzero((self.indeg > 0) & (self.indeg < heavy_min)))

    def row_class(self, v):
        r = self.label[v]
        return "heavy" if r < self.n_heavy else ("SELL" if r < self.n_heavy + self.n_sell else "zero")

    def bits(self, spare=0):
        """Magnitude bits of the integer values: a row's sum of |terms| stays below 2^52 (capped at 40 bits)."""
        return min(40, 52 - math.ceil(math.log2(int(self.indeg.max()) + 1))) - spare

    def reference(self, x, w=None):
        """Exact y = A^T x: every partial sum is a multiple of the terms' common grain below 2^53."""
        terms = x[self.f] if w is None else w * x[self.f]
        assert np.bincount(self.t, weights=np.abs(terms), minlength=self.n).max() < 2.0 ** 53
        return np.bincount(self.t, weights=terms, minlength=self.n)

    def check(self, y, want, what):
        if np.array_equal(y, want):
            return
        bad = np.flatnonzero(y != want)
        v = int(bad[0]) if len(bad) else int(np.flatnonzero(~(np.isnan(y) & np.isnan(want)))[0])
        pytest.fail(f"{what}: {len(bad)} rows differ; first: vertex {v}, label {self.label[v]}, {self.row_class(v)} row "
                    f"(in-degree {self.indeg[v]}): got {y[v]!r}, want {want[v]!r}", pytrace=False)


def int_values(n, bits, seed):
    """Integers of magnitude [2^(bits-1), 2^bits) with random signs, as doubles."""
    rng = np.random.default_rng(seed)
    mag = rng.integers(1 << (bits - 1), 1 << bits, n, dtype=np.int64)
    return (mag * rng.choice(np.array([-1, 1]), n)).astype(np.float64)


# ---- seam graphs: every class boundary inside a graph of a few thousand vertices -------------------------------------

SEAM_N = 4096
HEAVY_MIN, SEGMENT, TILE, TILE_CHUNK = 64, 32, 256, 8
BLOCK_FROM, BLOCK_LABELS, BLOCK_CHUNK = 1000, 400, 4
TABLE_LABELS = 128  # MGB200_SMEM_TABLE_KB=1
COMMON = {"MGB200_HEAVY_MIN_DEGREE": str(HEAVY_MIN), "MGB200_SMEM_TABLE_KB": "1", "MGB200_SELL_STAGE": "1",
          "MGB200_BLOCK_FROM": str(BLOCK_FROM), "MGB200_BLOCK_LABELS": str(BLOCK_LABELS),
          "MGB200_BLOCK_CHUNK": str(BLOCK_CHUNK)}
# tile_hot (131072 labels for 1 MB) is cut to block_from: the heavy rows' sources below 1000 are tiled, the rest blocked
SEAMS = {
    "tiles_blocks": {**COMMON, "MGB200_TILE_LABELS": str(TILE), "MGB200_TILE_HOT_MB": "1",
                     "MGB200_TILE_CHUNK": str(TILE_CHUNK)},
    "segments_blocks": {**COMMON, "MGB200_TILE_LABELS": "0", "MGB200_SEGMENT_EDGES": str(SEGMENT)},
    "segments": {**COMMON, "MGB200_TILE_LABELS": "0", "MGB200_BLOCK_LABELS": "0", "MGB200_SEGMENT_EDGES": str(SEGMENT)},
}
# exact in-degrees of the hub rows: both sides of the heavy threshold and of 2, 3, 4 and 8 cold segments
HUB_DEGREES = sorted({HEAVY_MIN - 1, HEAVY_MIN, HEAVY_MIN + 1} |
                     {k * SEGMENT + d for k in (2, 3, 4, 8) for d in (-1, 0, 1)} | {600})


def seam_graph(seed=0):
    """-> (n, f, t, hubs).  Every vertex has an edge into the coverage hub (heavy) and one into a SELL row, so every
    label is a source of both classes on both sides of every seam.  The hubs' in-degrees are exact (HUB_DEGREES); the
    SELL rows have in-degrees from 1 to 40 (slices of unequal width, so padding exists); a quarter of the vertices are
    zero rows.  Multi-edges and self-loops are part of it."""
    n = SEAM_N
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n)  # ids in no particular order
    cover, hubs = int(perm[0]), perm[1:1 + len(HUB_DEGREES)]
    sell = perm[1 + len(HUB_DEGREES):1 + len(HUB_DEGREES) + 3 * n // 4]
    f, t = [np.arange(n), np.arange(n)], [np.full(n, cover), rng.choice(sell, n)]
    for h, d in zip(hubs, HUB_DEGREES):
        src = rng.integers(0, n, d)  # with repeats: multi-edges
        src[0] = h  # a self-loop on a hub
        f.append(src)
        t.append(np.full(d, h))
    extra = rng.choice(sell, 4 * n, p=np.linspace(3.0, 0.1, len(sell)) / np.linspace(3.0, 0.1, len(sell)).sum())
    order = np.argsort(extra, kind="stable")
    first = np.r_[True, extra[order][1:] != extra[order][:-1]]
    occurrence = np.arange(len(extra)) - np.maximum.accumulate(np.where(first, np.arange(len(extra)), 0))
    extra = extra[np.sort(order[occurrence < 38])]  # at most 38 more per SELL row: every SELL row stays below 64
    f.append(rng.integers(0, n, len(extra)))
    t.append(extra)
    loops = sell[:50]
    f += [loops, sell[:200], sell[:200]]  # self-loops; 200 edges twice: multi-edges inside SELL rows
    t += [loops, sell[1:201], sell[1:201]]
    return n, np.concatenate(f).astype(np.uint64), np.concatenate(t).astype(np.uint64), hubs


def probe_labels():
    """Source labels on every seam of the tiles_blocks layout."""
    return {"first": 0, "last_table": TABLE_LABELS - 1, "first_after_table": TABLE_LABELS,
            "last_tiled": BLOCK_FROM - 1, "block_from": BLOCK_FROM, "end_of_first_block": BLOCK_FROM + BLOCK_LABELS - 1,
            "last": SEAM_N - 1}


def seam_claims(n, f, t, hubs):
    """What the seam tests rely on, from the host model alone."""
    m = Model(n, f, t, HEAVY_MIN)
    src, dst = m.label[m.f], m.label[m.t]
    deg = dict(zip(hubs.tolist(), m.indeg[hubs].tolist()))
    assert sorted(deg.values()) == HUB_DEGREES
    assert m.row_class(hubs[HUB_DEGREES.index(HEAVY_MIN - 1)]) == "SELL"
    assert all(m.row_class(h) == "heavy" for h, d in deg.items() if d >= HEAVY_MIN)
    assert m.n_heavy == 1 + sum(d >= HEAVY_MIN for d in HUB_DEGREES)  # the hubs and the coverage hub
    assert 0 < m.n_sell and m.n_heavy + m.n_sell < n  # zero rows exist
    heavy_in, sell_in = dst < m.n_heavy, (dst >= m.n_heavy) & (dst < m.n_heavy + m.n_sell)
    seams = ([TABLE_LABELS, BLOCK_FROM] + list(range(TILE, BLOCK_FROM, TILE)) +
             list(range(BLOCK_FROM + BLOCK_LABELS, n, BLOCK_LABELS)))
    for s in seams:
        for rows in (heavy_in, sell_in):
            assert np.any(rows & (src == s - 1)) and np.any(rows & (src == s)), s
    sell_deg = np.sort(m.indeg[m.vertex[m.n_heavy:m.n_heavy + m.n_sell]])[::-1]
    widths = sell_deg[::32]
    assert len(np.unique(widths)) > 5 and np.any(np.ptp(sell_deg[: len(sell_deg) // 32 * 32].reshape(-1, 32), axis=1) > 0)
    pairs = m.f * n + m.t
    assert len(np.unique(pairs)) < len(pairs) and np.any(m.f == m.t)  # multi-edges, self-loops
    assert np.any(m.f[heavy_in] == m.t[heavy_in]) and np.any(m.f[sell_in] == m.t[sell_in])
    for name, lab in probe_labels().items():
        v = m.vertex[lab]
        assert np.any(heavy_in & (m.f == v)) and np.any(sell_in & (m.f == v)), name
    # cold segments: in the `segments` layout every heavy edge is cold, so the hubs sit on both sides of k segments
    assert {k * SEGMENT + d for k in (2, 3, 4, 8) for d in (-1, 0, 1)} <= set(deg.values())
    return m


# ---- no GPU ------------------------------------------------------------------------------------------------------------


def test_label_model_matches_block_model_order():
    rng = np.random.default_rng(3)
    n = 3000
    f = rng.integers(0, n, 20000) // rng.integers(1, 4, 20000)  # skewed, with many ties in both degrees
    t = rng.integers(0, n, 20000) // rng.integers(1, 6, 20000)
    m = Model(n, f, t, heavy_min=20)
    want = sorted(range(n), key=lambda v: (-m.indeg[v], -m.outdeg[v], v))
    assert np.array_equal(m.vertex, want)
    bm = block_model(n, f, t, block_from=500, block_labels=300, heavy_min=20, sell_blocks=0)
    assert bm["heavy_rows"] == m.n_heavy > 0
    assert bm["heavy_edges"] == int(np.count_nonzero(m.label[m.t] < m.n_heavy))
    assert m.n_heavy + m.n_sell + int(np.count_nonzero(m.indeg == 0)) == n


def test_seam_graph_places_every_row_and_source():
    n, f, t, hubs = seam_graph()
    m = seam_claims(n, f, t, hubs)
    assert len(f) < 40 * n and int(m.indeg.max()) < 2 * n


def test_integer_values_are_wide_and_the_reference_exact():
    n, f, t, _ = seam_graph()
    m = Model(n, f, t, HEAVY_MIN)
    x = int_values(n, m.bits(), 1)
    assert np.all(np.abs(x) >= 2.0 ** 25) and np.any(x < 0) and np.any(x > 0)
    assert not np.array_equal(x.astype(np.float32).astype(np.float64), x)  # FP32 storage would lose bits
    exact = np.zeros(n, dtype=object)  # Python integers: no rounding at all
    np.add.at(exact, m.t, x[m.f].astype(np.int64).astype(object))
    assert np.array_equal(m.reference(x), exact.astype(np.float64))


# ---- GPU ---------------------------------------------------------------------------------------------------------------


def setenv(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def onehot_check(g, m, lab, what):
    """x = +inf at the source with label `lab`, 0 elsewhere: y is +inf exactly at its out-neighbours."""
    v = m.vertex[lab]
    x = np.zeros(m.n)
    x[v] = np.inf
    want = np.zeros(m.n)
    want[m.t[m.f == v]] = np.inf
    m.check(g.gather(x), want, f"{what}: one-hot at label {lab}")


@gpu
def test_default_layout_is_exact():
    """No knob set, RMAT scale 23 (MGB200_FULL_SCALE overrides it): tiles, blocks, staging (the vector is larger than
    L2) and the shared-memory table are all on."""
    import memgraph_b200 as mg
    scale = int(os.environ.get("MGB200_FULL_SCALE", "23"))
    n, e = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, e)
    m = Model(n, f, t)
    del f, t
    with mg.PageRankGraph.from_arrays(n, m.f.view(np.uint64), m.t.view(np.uint64)) as g:
        info = g.info
        for k in ("tiled_edges", "block_edges", "blocks", "stage_entries", "table_labels", "heavy_segments",
                  "sell_slices", "zero_rows"):
            assert info[k] > 0, k
        assert (info["heavy_rows"], info["sell_rows"]) == (m.n_heavy, m.n_sell)
        x = int_values(n, m.bits(), 11)
        m.check(g.gather(x), m.reference(x), f"RMAT-{scale}, default layout")
        table = info["table_labels"]
        for lab in (table - 1, table, 2 << 20, n - 1):
            onehot_check(g, m, lab, f"RMAT-{scale}, default layout")


# RMAT-18 under the variants table's layout, plus label blocks: with LAYOUT alone the graph lies below the default
# block_from and has no block passes, so nothing would be staged
SCALE = 18
BASE = {**LAYOUT, "MGB200_BLOCK_FROM": "131072", "MGB200_BLOCK_LABELS": "16384", "MGB200_SELL_STAGE": "1"}
# the same sums in the same order as BASE, so a float x gives BASE's bits too
SAME_ORDER = {**{k: (BASE, v) for k, v in VARIANTS.items()},
              "stage0": (BASE, {"MGB200_SELL_STAGE": "0"}),
              "idx_flags": (BASE, {"MGB200_IDX_FLAGS": "1"}),
              "build_chunks": (BASE, {"MGB200_BUILD_CHUNK_EDGES": "7777"})}
# other partials (tiles or blocks off, no block class at all): exact for integers only
OTHER_ORDER = {"tiles_off": (BASE, {"MGB200_TILE_LABELS": "0"}),
               "blocks_off": (BASE, {"MGB200_BLOCK_LABELS": "0"}),
               "layout_only": (LAYOUT, {})}


@pytest.fixture(scope="module")
def rmat18():
    import memgraph_b200 as mg
    n, e = 1 << SCALE, 16 << SCALE
    f, t = mg.rmat_edges_host(SCALE, e)
    m = Model(n, f, t, heavy_min=int(LAYOUT["MGB200_HEAVY_MIN_DEGREE"]))
    x = int_values(n, m.bits(), 5)
    xf = np.random.default_rng(6).standard_normal(n) * np.exp(np.random.default_rng(7).uniform(-20, 20, n))
    return {"model": m, "f": f, "t": t, "x": x, "want": m.reference(x), "xf": xf}


def gather_under(env, data, monkeypatch, *xs):
    import memgraph_b200 as mg
    setenv(monkeypatch, env)
    n = data["model"].n
    with mg.PageRankGraph.from_arrays(n, data["f"], data["t"]) as g:
        return g.info, [g.gather(x) for x in xs]


@pytest.fixture(scope="module")
def base_float(rmat18):
    """The float x gathered under BASE, and under LAYOUT: the multi-partition code path has no block class, so a
    variant that forces it keeps LAYOUT's partials."""
    out = {}
    for name, env in (("base", BASE), ("layout", LAYOUT)):
        with pytest.MonkeyPatch.context() as mp:
            info, (out[name],) = gather_under(env, rmat18, mp, rmat18["xf"])
        if name == "base":
            assert info["blocks"] > 1 and info["stage_entries"] > 0 and info["tiled_edges"] > 0
            assert info["table_labels"] > 0
    return out


@gpu
@pytest.mark.parametrize("name", list(SAME_ORDER))
def test_variant_is_exact_and_keeps_the_add_order(name, rmat18, base_float, monkeypatch):
    base, env = SAME_ORDER[name]
    info, (y, yf) = gather_under({**base, **env}, rmat18, monkeypatch, rmat18["x"], rmat18["xf"])
    rmat18["model"].check(y, rmat18["want"], f"RMAT-{SCALE}, {name}")
    same = "layout" if env.get("MGB200_FORCE_MULTI_PATH") == "1" else "base"
    assert (info["block_edges"] == 0) == (same == "layout")
    rmat18["model"].check(yf, base_float[same], f"RMAT-{SCALE}, {name}, float x against the {same} layout")


@gpu
@pytest.mark.parametrize("name", list(OTHER_ORDER))
def test_layout_change_is_exact(name, rmat18, monkeypatch):
    base, env = OTHER_ORDER[name]
    info, (y,) = gather_under({**base, **env}, rmat18, monkeypatch, rmat18["x"])
    if name == "tiles_off":
        assert info["tiled_edges"] == 0 and info["block_edges"] > 0
    elif name in ("blocks_off", "layout_only"):
        assert info["block_edges"] == 0 and info["stage_entries"] == 0
    rmat18["model"].check(y, rmat18["want"], f"RMAT-{SCALE}, {name}")


@pytest.fixture(scope="module")
def seam_data():
    n, f, t, hubs = seam_graph()
    return seam_claims(n, f, t, hubs)


@gpu
@pytest.mark.parametrize("layout", list(SEAMS))
def test_class_seams_are_exact(layout, seam_data, monkeypatch):
    import memgraph_b200 as mg
    m = seam_data
    setenv(monkeypatch, SEAMS[layout])
    with mg.PageRankGraph.from_arrays(m.n, m.f.astype(np.uint64), m.t.astype(np.uint64)) as g:
        info = g.info
        assert (info["heavy_rows"], info["sell_rows"]) == (m.n_heavy, m.n_sell)
        assert info["table_labels"] == TABLE_LABELS
        if layout == "tiles_blocks":
            assert info["tiled_edges"] + info["block_edges"] == info["heavy_edges"] and info["tiled_edges"] > 0
        if layout != "segments":
            assert info["blocks"] == -(-(m.n - BLOCK_FROM) // BLOCK_LABELS) and info["stage_entries"] > 0
        else:
            assert info["block_edges"] == info["tiled_edges"] == 0 and info["heavy_segments"] > m.n_heavy
        for seed in (1, 2):
            x = int_values(m.n, m.bits(), seed)
            m.check(g.gather(x), m.reference(x), f"seam graph, {layout}, seed {seed}")
        x = np.ones(m.n)  # small integers: the in-degrees themselves
        m.check(g.gather(x), m.indeg.astype(np.float64), f"seam graph, {layout}, in-degrees")


@gpu
@pytest.mark.parametrize("probe", list(probe_labels()))
def test_one_hot_probe_reaches_only_its_out_neighbours(probe, seam_data, monkeypatch):
    import memgraph_b200 as mg
    m = seam_data
    setenv(monkeypatch, SEAMS["tiles_blocks"])
    with mg.PageRankGraph.from_arrays(m.n, m.f.astype(np.uint64), m.t.astype(np.uint64)) as g:
        onehot_check(g, m, probe_labels()[probe], f"seam graph, tiles_blocks, {probe}")


@gpu
def test_weighted_handle_is_exact(rmat18, monkeypatch):
    import memgraph_b200 as mg
    from memgraph_b200 import personalized as P
    setenv(monkeypatch, BASE)
    m = rmat18["model"]
    w = dyadic_weights(len(m.f))
    x = int_values(m.n, m.bits(spare=4), 9)  # |w| < 4 and w a multiple of 1/4: two more bits each side
    with P.weighted_graph(m.n, rmat18["f"], rmat18["t"], w) as g:
        m.check(g.gather(x, weighted=True), m.reference(x, w), f"RMAT-{SCALE}, weighted")
        m.check(g.gather(x), m.reference(x), f"RMAT-{SCALE}, weighted handle, weighted=False")
    with mg.PageRankGraph.from_arrays(m.n, rmat18["f"], rmat18["t"]) as g:
        with pytest.raises(mg.MgB200Error, match="no edge weights"):
            g.gather(x, weighted=True)


def gamma(k):
    return k * U / (1 - k * U)


@gpu
def test_float_values_meet_the_summation_bound_and_repeat(rmat18, base_float, monkeypatch):
    """Random FP64 values of mixed sign over about 58 binades: every heavy row and 10^4 SELL rows within
    gamma_(d+s) * sum |terms| of the exact sum, where d is the row's in-degree and s <= d its partial count."""
    import memgraph_b200 as mg
    m, xf = rmat18["model"], rmat18["xf"]
    setenv(monkeypatch, BASE)
    with mg.PageRankGraph.from_arrays(m.n, rmat18["f"], rmat18["t"]) as g:
        y1, y2 = g.gather(xf), g.gather(xf)
    assert np.array_equal(y1, y2) and np.array_equal(y1, base_float["base"])
    order = np.argsort(m.label[m.t], kind="stable")
    terms = xf[m.f][order]
    first = np.r_[0, np.cumsum(np.bincount(m.label[m.t], minlength=m.n))]
    rng = np.random.default_rng(10)
    rows = np.r_[np.arange(m.n_heavy), rng.choice(np.arange(m.n_heavy, m.n_heavy + m.n_sell), 10000, replace=False)]
    for r in rows:
        tr = terms[first[r]:first[r + 1]]
        exact = math.fsum(tr)
        d = len(tr)
        bound = gamma(2 * d) * float(np.abs(tr).sum()) + U * abs(exact)
        v = m.vertex[r]
        assert abs(y1[v] - exact) <= bound, (int(v), int(r), m.row_class(v), d, y1[v], exact)


@gpu
def test_gather_leaves_the_handle_as_a_fresh_one(rmat18, monkeypatch):
    """run, Katz and cuGraph PageRank after a gather on the same handle equal their runs on a fresh handle."""
    import memgraph_b200 as mg
    from memgraph_b200 import katz
    from memgraph_b200 import personalized as P
    setenv(monkeypatch, BASE)
    m, n = rmat18["model"], rmat18["model"].n
    alpha = katz_alpha(rmat18["f"], n)
    algos = {"pagerank": lambda g: g.run(max_iterations=20, stop_epsilon=0.0)[0],
             "katz": lambda g: katz.set_katz(g, alpha=alpha, epsilon=1e-3)[0],
             "cugraph": lambda g: P.cugraph_pagerank(g, np.array([0, 12345]), np.array([0.4, 0.6]), max_iterations=30,
                                                     stop_epsilon=0.0)[0]}
    with mg.PageRankGraph.from_arrays(n, rmat18["f"], rmat18["t"]) as used:
        for name, algo in algos.items():
            used.gather(rmat18["xf"])
            got = algo(used)
            with mg.PageRankGraph.from_arrays(n, rmat18["f"], rmat18["t"]) as fresh:
                want = algo(fresh)
            assert np.array_equal(got, want), name
        m.check(used.gather(rmat18["x"]), rmat18["want"], f"RMAT-{SCALE}, gather after the algorithms")


@gpu
def test_empty_graphs_and_bad_arguments():
    import memgraph_b200 as mg
    with mg.PageRankGraph.from_arrays(0, [], []) as g:
        assert g.gather(np.zeros(0)).shape == (0,)
    with mg.PageRankGraph.from_arrays(7, [], []) as g:
        assert np.array_equal(g.gather(np.arange(7.0) + 1), np.zeros(7))
        with pytest.raises(mg.MgB200Error, match="x must hold 7 values"):
            g.gather(np.zeros(6))
    with mg.PageRankGraph.from_arrays(3, [0, 1, 2, 2], [1, 2, 0, 2]) as g:
        assert np.array_equal(g.gather(np.array([1.0, 2.0, 4.0])), np.array([4.0, 1.0, 6.0]))


def partitioned_case():
    """Child: a gather on either partition of a two-partition graph on device 0 is refused."""
    import memgraph_b200 as mg
    rng = np.random.default_rng(8)
    n = 3000
    f, t = rng.integers(0, n, 20000), rng.integers(0, n, 20000)
    graphs = [mg.PageRankGraph.from_arrays(n, f, t, device=0, part_rank=q, part_world=2) for q in range(2)]
    for g in graphs:
        with pytest.raises(mg.MgB200Error, match="single-partition"):
            g.gather(np.ones(n))
        g.close()


@gpu
def test_partitioned_handle_is_refused():
    from test_gpu_partitions_one_device import in_child
    in_child(partitioned_case)

"""Weighted shortest paths on the GPU (memgraph_b200/csrc/wsp.cu through memgraph_b200.bfs) against the cursor
restatement oracle/wsp_oracle.c: total_weight bit for bit and hops exactly, from the reference's fixtures up to RMAT
scale-20, plus the unit-weight agreement with gpu_bfs, determinism, and the reported invalid edge."""
import math

import numpy as np
import pytest

import memgraph_b200 as mg
from memgraph_b200 import bfs
from test_wsp_oracle import fixture_arrays, fixture_cases, oracle_wsp, random_graph, same_bits

pytestmark = pytest.mark.gpu

RUN_KEYS = ("rounds", "buckets", "hop_levels", "delta", "reached", "relaxations", "entries_inspected", "invalid_edge",
            "kernel_launches")


def gpu_wsp(n, f, t, w, source, direction=0, upper_bound=None):
    with bfs.BfsGraph(n, f, t) as g:
        g.set_weights(f, t, w)
        return g.weighted_distances(source, direction, upper_bound)


def check(n, f, t, w, source, direction, upper_bound, ctx):
    rc, dist, depth, hops, invalid = oracle_wsp(n, f, t, w, source, direction, upper_bound)
    if rc == 3:
        with pytest.raises(bfs.InvalidWeight) as err:
            gpu_wsp(n, f, t, w, source, direction, upper_bound)
        assert err.value.edge_index == invalid, ctx
        return None
    assert rc == 0, ctx
    gd, gh, stats = gpu_wsp(n, f, t, w, source, direction, upper_bound)
    assert same_bits(gd, dist), ctx
    assert np.array_equal(gh, hops), ctx
    assert stats["reached"] == int((hops >= 0).sum()), ctx
    return stats


def test_reference_fixtures():
    for case in fixture_cases():
        f, t, w = fixture_arrays(case)
        ub = case["upper_bound"]
        if ub is not None and ub < 1:
            with bfs.BfsGraph(case["n"], f, t) as g:
                g.set_weights(f, t, w)
                with pytest.raises(mg.MgB200Error, match="must be at least 1"):
                    g.weighted_distances(case["start"], case["direction"], ub)
            continue
        check(case["n"], f, t, w, case["start"], case["direction"], ub, case["name"])
        if "rows" in case:
            dist, hops, _ = gpu_wsp(case["n"], f, t, w, case["start"], case["direction"], ub)
            for v, total, size in case["rows"]:
                assert dist[v] == total and (size is None or hops[v] == size), case["name"]


def test_random_multigraphs():
    rng = np.random.default_rng(77)
    errors = 0
    for i in range(300):
        n, f, t, w = random_graph(rng)
        ub = [None, 1, 2, 3, 5][i % 5]
        errors += check(n, f, t, w, int(rng.integers(0, n)), i % 3, ub, (i, n, f.tolist(), t.tolist(), w.tolist())) \
            is None
    assert 5 <= errors <= 150


@pytest.mark.parametrize("scale", [16, 20])
def test_rmat(scale):
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    for kind in ("uniform", "int"):
        w = bfs.splitmix_weights(m, kind)
        with bfs.BfsGraph(n, f, t) as g:
            g.set_weights(f, t, w)
            source = int(np.bincount(f.astype(np.int64), minlength=n).argmax())  # a hub: the largest frontier
            for direction in (0, 1, 2):
                for ub in (1, 2, 3, None):
                    rc, dist, _, hops, _ = oracle_wsp(n, f, t, w, source, direction, ub)
                    assert rc == 0
                    gd, gh, stats = g.weighted_distances(source, direction, ub)
                    ctx = (scale, kind, direction, ub)
                    assert same_bits(gd, dist), ctx
                    assert np.array_equal(gh, hops), ctx
                    assert stats["reached"] > 0 and stats["invalid_edge"] == 2**64 - 1, ctx


def test_long_path_stars_isolated_source_and_infinity():
    n = 100_000  # a weighted path 0 -> 1 -> ... walked by 10^5 passes
    f, t = np.arange(n - 1), np.arange(1, n)
    w = bfs.splitmix_weights(n - 1)
    for direction, ub in [(0, None), (2, None), (0, 50_000)]:
        check(n, f, t, w, 0, direction, ub, ("path", direction, ub))
    for deg in (5_000, 300_000):  # a hub list cut over many warps
        n = deg + 1
        f, t = np.zeros(deg, dtype=np.int64), np.arange(1, n)
        w = bfs.splitmix_weights(deg, "int")
        for direction in (0, 1, 2):
            check(n, f, t, w, 0, direction, None, ("star out", deg, direction))
            check(n, t, f, w, 0, direction, 2, ("star in", deg, direction))
            check(n, f, t, w, 7, direction, None, ("leaf", deg, direction))
    dist, hops, stats = gpu_wsp(4, [1, 2], [2, 3], [1.0, 1.0], 0)
    assert np.isnan(dist).all() and (hops == -1).all() and stats["reached"] == 0
    f, t = [0, 1, 0, 2, 3], [1, 2, 2, 3, 0]
    w = [math.inf, 0.0, math.inf, 1.0, 0.0]
    for ub in (None, 1, 2, 3):
        check(4, f, t, w, 0, 0, ub, ("inf", ub))
    dist, hops, _ = gpu_wsp(4, f, t, w, 0)
    assert dist[1:].tolist() == [math.inf] * 3 and hops[1:].tolist() == [1, 1, 2]


def test_unit_weights_agree_with_bfs():
    scale = 16
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    with bfs.BfsGraph(n, f, t) as g:
        g.set_weights(f, t, np.ones(m))
        for direction in (0, 1, 2):
            depth, _ = g.distances(0, direction)
            dist, hops, _ = g.weighted_distances(0, direction)
            assert np.array_equal(hops, depth), direction
            assert np.array_equal(np.where(depth >= 0, depth.astype(np.float64), np.nan), dist, equal_nan=True)
            for ub in (1, 2, 3):
                bounded_depth, _ = g.distances(0, direction, 1, ub)
                d2, h2, _ = g.weighted_distances(0, direction, ub)
                assert np.array_equal(h2 >= 0, bounded_depth >= 0), (direction, ub)
                assert np.array_equal(h2, bounded_depth), (direction, ub)


def test_two_runs_are_identical_and_the_smallest_invalid_edge_is_reported():
    scale = 18
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    w = bfs.splitmix_weights(m)
    with bfs.BfsGraph(n, f, t) as g:
        g.set_weights(f, t, w)
        for direction, ub in [(0, None), (2, None), (1, 3)]:
            a = g.weighted_distances(0, direction, ub)
            b = g.weighted_distances(0, direction, ub)
            assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
            assert [a[2][k] for k in RUN_KEYS] == [b[2][k] for k in RUN_KEYS]
        assert a[2]["buckets"] == 0 and a[2]["rounds"] <= 3
    # invalid weights scattered over the graph: the reported index is the oracle's smallest evaluated one
    rng = np.random.default_rng(3)
    w = bfs.splitmix_weights(m)
    bad = rng.choice(m, size=50, replace=False)
    w[bad[:25]] = -1.0
    w[bad[25:]] = math.nan
    source = int(f[bad.min()])  # certainly evaluated from here
    for direction, ub in [(0, None), (1, None), (2, 2), (0, 1)]:
        check(n, f, t, w, source, direction, ub, ("invalid", direction, ub))
    # an invalid entry that is never evaluated changes nothing
    w2 = np.ones(5)
    w2[4] = -1.0
    dist, hops, _ = gpu_wsp(6, [0, 1, 2, 3, 4], [1, 2, 3, 4, 5], w2, 0, 0, 3)
    assert hops.tolist() == [-1, 1, 2, 3, -1, -1]
    with pytest.raises(bfs.InvalidWeight) as err:
        gpu_wsp(6, [0, 1, 2, 3, 4], [1, 2, 3, 4, 5], w2, 0, 0, 5)
    assert err.value.edge_index == 4


def test_one_shot_entry_point():
    dist, hops = bfs.weighted_shortest_paths(3, [0, 1], [1, 2], [0.5, 0.25], 0)
    assert math.isnan(dist[0]) and dist[1:].tolist() == [0.5, 0.75] and hops.tolist() == [-1, 1, 2]


def test_set_weights_refuses_other_pairs_and_leaves_no_weights_behind():
    f, t = np.array([0, 1, 2, 2]), np.array([1, 2, 0, 3])
    with bfs.BfsGraph(4, f, t) as g:
        g.set_weights(f, t, [1.0, 2.0, 3.0, 4.0])
        assert g.weighted_distances(0)[0][1:].tolist() == [1.0, 3.0, 7.0]
        g.set_weights(f[::-1], t[::-1], [1.0, 2.0, 3.0, 4.0])  # the same pairs in another order, other weights
        assert g.weighted_distances(0)[0][1:].tolist() == [4.0, 7.0, 8.0]
        for bad_f, bad_t in [([0, 1, 2, 3], [1, 2, 0, 2]), ([0, 1, 2, 2], [1, 2, 0, 0]), ([1, 1, 2, 2], [0, 2, 0, 3])]:
            with pytest.raises(mg.MgB200Error, match="pairs differ from the graph's"):
                g.set_weights(bad_f, bad_t, [1.0, 1.0, 1.0, 1.0])
            with pytest.raises(mg.MgB200Error, match="has no weights"):
                g.weighted_distances(0, 1)  # neither list keeps weights after a refused call
        g.set_weights(f, t, [1.0, 2.0, 3.0, 4.0])
        assert g.weighted_distances(0, 2)[0][1:].tolist() == [1.0, 3.0, 3.0 + 4.0]

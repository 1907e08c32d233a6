"""Strongly connected components on the device (memgraph_b200/csrc/scc.cu) against oracle/scc_oracle.c, which
tests/test_scc_oracle.py pins to networkx.  The output is integers: every case is np.array_equal, and two runs, the
one-shot and the resident path give byte-identical outputs and stats (run_ms aside)."""
import ctypes

import numpy as np
import pytest

from _checkers import oracle_rmat_edges
from test_scc_oracle import block_chain, oracle_scc

pytestmark = pytest.mark.gpu

K_NARROW = 1024        # scc.cu: kNarrow, the largest frontier one CTA expands
K_THREAD_ENTRIES = 16  # undirected_walk.cuh: a thread walks a list up to this long, a warp up to K_WARP_ENTRIES
K_WARP_ENTRIES = 4096


@pytest.fixture(scope="module")
def cc():
    from memgraph_b200 import connectivity
    return connectivity


def same_stats(a, b):
    return {k: v for k, v in a.items() if k != "run_ms"} == {k: v for k, v in b.items() if k != "run_ms"}


def check(cc, n, f, t):
    """One-shot and resident runs equal the oracle and each other; two runs are byte-identical; the stats agree."""
    f = np.asarray(f, dtype=np.uint64)
    t = np.asarray(t, dtype=np.uint64)
    exp = oracle_scc(n, f, t)
    got = cc.strongly_connected_components(n, f, t)
    assert np.array_equal(got, exp)
    with cc.BfsGraph(n, f, t) as g:
        first, stats = cc.scc_run(g)
        second, again = cc.scc_run(g)
    assert first.tobytes() == second.tobytes() == got.tobytes()
    assert same_stats(stats, again), (stats, again)
    if n:
        sizes = np.bincount(got)
        assert stats["components"] == got.max() + 1
        assert stats["largest_component"] == sizes.max()
        assert stats["trimmed"] <= (sizes == 1).sum()
        assert stats["pivot_component"] == 0 or stats["pivot_component"] in set(sizes.tolist())
    else:
        assert stats["components"] == 0 and stats["largest_component"] == 0 and stats["kernel_launches"] == 0
    return stats


def test_small_sizes(cc):
    rng = np.random.default_rng(1)
    for n in (0, 1, 2, 31, 32, 33):
        for m in (0, n // 2, 2 * n):
            check(cc, n, rng.integers(0, max(n, 1), m), rng.integers(0, max(n, 1), m))


def test_self_loops_multi_edges_and_two_cycles(cc):
    n = 1000
    v = np.arange(n)
    stats = check(cc, n, v, v)  # self-loops only: every vertex alone, all trimmed
    assert stats["components"] == n and stats["trimmed"] == n
    stats = check(cc, n, np.concatenate([v[0::2], v[1::2]]), np.concatenate([v[1::2], v[0::2]]))  # 2-cycles
    assert stats["components"] == n // 2 and stats["largest_component"] == 2
    rng = np.random.default_rng(2)
    f, t = rng.integers(0, n, 1500), rng.integers(0, n, 1500)
    single = check(cc, n, f, t)
    multi = check(cc, n, np.concatenate([f, f, f, v]), np.concatenate([t, t, t, v]))  # repeated, plus self-loops
    assert multi["components"] == single["components"]


@pytest.mark.parametrize("n,m", [(1000, 600), (50_000, 40_000), (200_000, 300_000)])
def test_symmetric_edge_sets_equal_wcc(cc, n, m):
    rng = np.random.default_rng(n)
    f, t = rng.integers(0, n, m), rng.integers(0, n, m)
    f, t = np.concatenate([f, t]), np.concatenate([t, f])
    check(cc, n, f, t)
    with cc.BfsGraph(n, f.astype(np.uint64), t.astype(np.uint64)) as g:
        strong, _ = cc.scc_run(g)
        weak, _ = cc.wcc_run(g)
    assert np.array_equal(strong, weak)


def test_dag_with_shuffled_ids_is_all_trimmed(cc):
    n = 100_000
    rng = np.random.default_rng(3)
    a, b = rng.integers(0, n, 4 * n), rng.integers(0, n, 4 * n)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    keep = lo != hi
    perm = rng.permutation(n)
    stats = check(cc, n, perm[lo[keep]], perm[hi[keep]])
    assert stats["trimmed"] == n and stats["components"] == n
    assert stats["pivot_component"] == 0 and stats["coloring_rounds"] == 0 and stats["levels"] == 0


def test_long_paths_and_cycles_in_shuffled_order(cc):
    n = 100_000
    perm = np.random.default_rng(4).permutation(n)
    stats = check(cc, n, perm[:-1], perm[1:])  # a path: trimmed, the chain followed by one thread per end
    assert stats["trimmed"] == n
    stats = check(cc, n, perm, np.roll(perm, -1))  # a cycle: one component, found by forward-backward
    assert stats["components"] == 1 and stats["pivot_component"] == n and stats["trimmed"] == 0
    assert stats["levels"] >= 2 * n - 2
    assert stats["host_round_trips"] < 0.01 * stats["levels"]
    # a cycle beside a path
    stats = check(cc, n, np.concatenate([perm[:50_000], perm[50_000:-1]]),
                  np.concatenate([np.roll(perm[:50_000], -1), perm[50_001:]]))
    assert stats["largest_component"] == 50_000


@pytest.mark.parametrize("leaves", [K_THREAD_ENTRIES, K_THREAD_ENTRIES + 1, K_WARP_ENTRIES, K_WARP_ENTRIES + 1, 300_000])
def test_stars_across_the_walk_thresholds(cc, leaves):
    n = leaves + 1
    hub = np.zeros(leaves, dtype=np.int64)
    tips = np.arange(1, n)
    check(cc, n, tips, hub)  # in-star
    check(cc, n, hub, tips)  # out-star
    stats = check(cc, n, np.concatenate([hub, tips]), np.concatenate([tips, hub]))  # two-way: one component
    assert stats["components"] == 1 and stats["pivot_component"] == n
    # the hub is the largest id and points into a cycle of the leaves
    ring = np.arange(leaves)
    stats = check(cc, n, np.concatenate([[leaves], ring]), np.concatenate([[0], np.roll(ring, -1)]))
    assert stats["largest_component"] == leaves


@pytest.mark.parametrize("width", [K_NARROW, K_NARROW + 1])
def test_frontiers_at_the_narrow_threshold(cc, width):
    """A source fans out to `width` vertices, which all lead back to it through a sink: the second level of each search
    is exactly `width` vertices wide."""
    n = width + 2
    src, sink = 0, n - 1
    mid = np.arange(1, width + 1)
    f = np.concatenate([np.zeros(width, dtype=np.int64), mid, [sink]])
    t = np.concatenate([mid, np.full(width, sink), [src]])
    perm = np.random.default_rng(width).permutation(n)
    stats = check(cc, n, perm[f], perm[t])
    assert stats["components"] == 1 and stats["pivot_component"] == n


@pytest.mark.parametrize("blocks,ascending", [(300, False), (300, True)])
def test_chains_of_blocks(cc, blocks, ascending):
    n, f, t = block_chain(blocks, 4, np.random.default_rng(blocks), ascending)
    stats = check(cc, n, f, t)
    assert stats["components"] == blocks and stats["largest_component"] == 4
    assert stats["coloring_rounds"] >= 1


def test_random_dag_of_blocks(cc):
    rng = np.random.default_rng(5)
    blocks = 1 << 14
    sizes = rng.integers(1, 65, blocks)
    start = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    n = int(sizes.sum())
    f, t = [], []
    for s, k in zip(start, sizes):  # each block a cycle (a singleton has no edge of its own)
        if k > 1:
            f.append(np.arange(s, s + k))
            t.append(np.roll(np.arange(s, s + k), -1))
    a, b = rng.integers(0, blocks, 3 * blocks), rng.integers(0, blocks, 3 * blocks)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    keep = lo != hi  # block edges go from a lower block to a higher one: a DAG of blocks
    f.append(start[lo[keep]] + rng.integers(0, 64, keep.sum()) % sizes[lo[keep]])
    t.append(start[hi[keep]] + rng.integers(0, 64, keep.sum()) % sizes[hi[keep]])
    perm = rng.permutation(n)
    stats = check(cc, n, perm[np.concatenate(f)], perm[np.concatenate(t)])
    assert stats["components"] == blocks


def test_pivot_tie_and_a_giant_without_vertex_zero(cc):
    # two disjoint 3-cycles with equal in * out products: the pivot is the smaller id
    stats = check(cc, 6, [3, 4, 5, 0, 1, 2], [4, 5, 3, 1, 2, 0])
    assert stats["pivot_component"] == 3 and stats["coloring_rounds"] == 1
    rng = np.random.default_rng(6)
    n = 200_000
    f, t = rng.integers(1000, n, 4 * n), rng.integers(1000, n, 4 * n)  # the giant lives in 1000..
    f = np.concatenate([f, np.arange(0, 1000, 2), np.arange(1, 1000, 2)])  # 0..999: 2-cycles
    t = np.concatenate([t, np.arange(1, 1000, 2), np.arange(0, 1000, 2)])
    stats = check(cc, n, f, t)
    got = cc.strongly_connected_components(n, f, t)
    assert got[0] == got[1] == 0 and np.bincount(got).argmax() >= 500
    assert stats["pivot_component"] == stats["largest_component"]


@pytest.mark.parametrize("ratio", [1.0, 1.2, 2.0])
def test_erdos_renyi(cc, ratio):
    n = 1 << 20
    m = int(ratio * n)
    rng = np.random.default_rng(int(10 * ratio))
    check(cc, n, rng.integers(0, n, m), rng.integers(0, n, m))


@pytest.mark.parametrize("scale", [20, 22])
def test_rmat(cc, scale):
    n = 1 << scale
    f, t = oracle_rmat_edges(scale)
    stats = check(cc, n, f, t)
    if scale == 20:  # a full trim leaves only the giant component
        assert stats["trimmed"] + stats["pivot_component"] == n
        assert stats["coloring_rounds"] == 0


def test_should_abort(cc):
    from memgraph_b200 import _native as N
    from memgraph_b200.pagerank import MgB200Error
    n = 10_000
    perm = np.random.default_rng(7).permutation(n)
    calls = []
    with cc.BfsGraph(n, perm, np.roll(perm, -1)) as g:
        with pytest.raises(MgB200Error) as e:
            cc.scc_run(g, should_abort=lambda: calls.append(1) or len(calls) > 2)
        assert e.value.code == N.ERR_ABORTED
        assert len(calls) == 3
        got, stats = cc.scc_run(g, should_abort=lambda: False)
    assert not got.any() and stats["components"] == 1
    # component_out is left untouched
    out = np.full(n, 7, dtype=np.int64)
    with cc.BfsGraph(n, perm, np.roll(perm, -1)) as g:
        rc = N.lib().mgb200_scc_run(g._h, N.ABORT_FN(lambda _u: 1), None, out.ctypes.data, None)
    assert rc == N.ERR_ABORTED and (out == 7).all()


def test_argument_errors(cc):
    from memgraph_b200 import _native as N
    lib = N.lib()
    s = np.array([0, 1], dtype=np.uint64)
    assert lib.mgb200_strongly_connected_components(3, 2, s.ctypes.data, s.ctypes.data, None) == N.ERR_INVALID_ARGUMENT
    assert lib.mgb200_scc_run(None, N.ABORT_FN(), None, None, None) == N.ERR_INVALID_ARGUMENT
    assert lib.mgb200_strongly_connected_components(0, 0, None, None, None) == N.OK
    with cc.BfsGraph(3, s, s + 1) as g:
        assert lib.mgb200_scc_run(g._h, N.ABORT_FN(), None, None, None) == N.ERR_INVALID_ARGUMENT
        out = np.zeros(3, dtype=np.int64)
        assert lib.mgb200_scc_run(g._h, N.ABORT_FN(), None, out.ctypes.data, None) == N.OK  # stats may be null
        assert out.tolist() == [0, 1, 2]
    st = N.SccStats()
    with cc.BfsGraph(0, [], []) as g:
        assert lib.mgb200_scc_run(g._h, N.ABORT_FN(), None, None, ctypes.byref(st)) == N.OK
        assert st.components == 0 and st.kernel_launches == 0


def test_wcc_scc_and_bfs_share_one_handle(cc):
    from test_wcc_oracle import oracle_wcc
    scale = 18
    n = 1 << scale
    f, t = oracle_rmat_edges(scale)
    with cc.BfsGraph(n, f, t) as g:
        bfs_before, _ = g.distances(0)
        wcc_before, _ = cc.wcc_run(g)
        scc, _ = cc.scc_run(g)
        wcc_after, _ = cc.wcc_run(g)
        bfs_after, _ = g.distances(0)
        scc_again, _ = cc.scc_run(g)
    assert np.array_equal(scc, oracle_scc(n, f, t)) and scc.tobytes() == scc_again.tobytes()
    assert np.array_equal(wcc_before, oracle_wcc(n, f, t)) and wcc_before.tobytes() == wcc_after.tobytes()
    assert bfs_before.tobytes() == bfs_after.tobytes()

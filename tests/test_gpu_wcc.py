"""Weakly connected components on the device (memgraph_b200/csrc/wcc.cu) against oracle/wcc_oracle.c, which
tests/test_wcc_oracle.py pins to the reference's own module.  The output is integers: every case is np.array_equal."""
import numpy as np
import pytest

from _checkers import oracle_rmat_edges
from test_wcc_oracle import e2e_steps, oracle_wcc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cc():
    from memgraph_b200 import connectivity
    return connectivity


def check(cc, n, f, t):
    """One-shot and resident runs equal the oracle and each other; two runs are byte-identical; the stats agree."""
    f = np.asarray(f, dtype=np.uint64)
    t = np.asarray(t, dtype=np.uint64)
    exp = oracle_wcc(n, f, t)
    got = cc.weakly_connected_components(n, f, t)
    assert np.array_equal(got, exp)
    with cc.BfsGraph(n, f, t) as g:
        first, stats = cc.wcc_run(g)
        second, _ = cc.wcc_run(g)
    assert first.tobytes() == second.tobytes() == got.tobytes()
    if n:
        assert stats["components"] == got.max() + 1
        assert stats["largest_component"] == np.bincount(got).max()
    else:
        assert stats["components"] == 0 and stats["largest_component"] == 0
    return stats


def test_e2e_fixtures(cc):
    for name, nodes, edges, expected in e2e_steps():
        e = np.array(edges, dtype=np.int64).reshape(-1, 2)
        got = cc.weakly_connected_components(len(nodes), e[:, 0], e[:, 1])
        assert sorted(zip(nodes, got.tolist())) == expected, name


def test_small_sizes(cc):
    rng = np.random.default_rng(1)
    for n in (0, 1, 2, 31, 32, 33):
        for m in (0, n // 2, 2 * n):
            check(cc, n, rng.integers(0, max(n, 1), m), rng.integers(0, max(n, 1), m))


def test_isolated_self_loops_and_multi_edges(cc):
    n = 1000
    stats = check(cc, n, [], [])
    assert stats["components"] == n and stats["largest_component"] == 1
    v = np.arange(n)
    stats = check(cc, n, v, v)  # self-loops only
    assert stats["components"] == n
    rng = np.random.default_rng(2)
    f, t = rng.integers(0, n, 300), rng.integers(0, n, 300)
    single = check(cc, n, f, t)
    multi = check(cc, n, np.concatenate([f, f, t, f]), np.concatenate([t, t, f, t]))  # both directions, repeated
    assert multi["components"] == single["components"]


def test_long_paths_in_shuffled_id_order(cc):
    n = 100_000
    perm = np.random.default_rng(3).permutation(n)
    stats = check(cc, n, perm[:-1], perm[1:])  # u -> v along the path
    assert stats["components"] == 1
    check(cc, n, perm[1:], perm[:-1])  # and the other direction
    check(cc, n, np.concatenate([perm[:50_000 - 1], perm[50_001:]]), np.concatenate([perm[1:50_000], perm[50_000:-1]]))


def test_stars(cc):
    n = 300_000  # the hub's list crosses the one-block-per-vertex threshold
    leaves = np.arange(1, n)
    hub = np.full(n - 1, 0)
    check(cc, n, leaves, hub)  # in-star
    check(cc, n, hub, leaves)  # out-star
    hub = np.full(n // 2, n - 1)  # the hub is the largest id: every leaf's root is hooked under a smaller one
    check(cc, n, hub, np.arange(n // 2))
    check(cc, n, np.arange(n // 2), hub)


def test_many_small_components_no_giant(cc):
    n = 1_000_000
    rng = np.random.default_rng(4)
    stats = check(cc, n, rng.integers(0, n, n // 4), rng.integers(0, n, n // 4))
    assert stats["largest_component"] < 100


def test_giant_component_excludes_vertex_zero(cc):
    rng = np.random.default_rng(5)
    n = 200_000
    f = rng.integers(1000, n, 4 * n)  # vertices 1000.. form the giant; 0..999 are pairs and singletons
    t = rng.integers(1000, n, 4 * n)
    f = np.concatenate([f, np.arange(0, 1000, 2)])
    t = np.concatenate([t, np.arange(1, 1000, 2)])
    stats = check(cc, n, f, t)
    got = cc.weakly_connected_components(n, f, t)
    assert got[0] == 0 and got[1] == 0 and np.bincount(got).argmax() >= 500
    assert stats["skipped_vertices"] > n // 2


@pytest.mark.parametrize("n,m", [(5000, 2500), (5000, 5000), (5000, 20000), (200_000, 150_000), (200_000, 800_000)])
def test_erdos_renyi(cc, n, m):
    rng = np.random.default_rng(n + m)
    check(cc, n, rng.integers(0, n, m), rng.integers(0, n, m))


@pytest.mark.parametrize("scale", [20, 22])
def test_rmat(cc, scale):
    n = 1 << scale
    f, t = oracle_rmat_edges(scale)
    stats = check(cc, n, f, t)
    assert stats["skipped_vertices"] > 0
    if scale == 20:
        assert stats["edges_inspected"] < 2 * len(f)  # the giant component's lists were skipped


def test_argument_errors(cc):
    import ctypes
    from memgraph_b200 import _native as N
    lib = N.lib()
    s = np.array([0, 1], dtype=np.uint64)
    assert lib.mgb200_weakly_connected_components(3, 2, s.ctypes.data, s.ctypes.data, None) == N.ERR_INVALID_ARGUMENT
    assert lib.mgb200_wcc_run(None, None, None) == N.ERR_INVALID_ARGUMENT
    assert lib.mgb200_weakly_connected_components(0, 0, None, None, None) == N.OK
    with cc.BfsGraph(3, s, s + 1) as g:
        assert lib.mgb200_wcc_run(g._h, None, None) == N.ERR_INVALID_ARGUMENT
        out = np.zeros(3, dtype=np.int64)
        assert lib.mgb200_wcc_run(g._h, out.ctypes.data, None) == N.OK  # stats may be null
        assert out.tolist() == [0, 0, 0]
    st = N.WccStats()
    with cc.BfsGraph(0, [], []) as g:
        assert lib.mgb200_wcc_run(g._h, None, ctypes.byref(st)) == N.OK
        assert st.components == 0 and st.kernel_launches == 0

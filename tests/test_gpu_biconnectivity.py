"""Bridges and biconnected components on the device (memgraph_b200/csrc/biconnectivity.cu) against
oracle/biconnectivity_oracle.c, which tests/test_biconnectivity_oracle.py pins to the reference's own modules.  The
output is integers with the same first-edge numbering: every case is np.array_equal."""
import numpy as np
import pytest

from _checkers import oracle_rmat_edges
from test_biconnectivity_oracle import oracle_biconnectivity

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cc():
    from memgraph_b200 import connectivity
    return connectivity


def check(cc, n, f, t):
    """One-shot and resident runs equal the oracle and each other; two runs are byte-identical, stats included; the
    stats agree with the outputs."""
    f = np.asarray(f, dtype=np.uint64)
    t = np.asarray(t, dtype=np.uint64)
    exp_bridge, exp_bcc = oracle_biconnectivity(n, f, t)
    with cc.BfsGraph(n, f, t) as g:
        bridge, bcc, stats = cc.biconnectivity_run(g, f, t)
        bridge2, bcc2, stats2 = cc.biconnectivity_run(g, f, t)
    assert np.array_equal(bridge, exp_bridge)
    assert np.array_equal(bcc, exp_bcc)
    assert bridge.tobytes() == bridge2.tobytes() and bcc.tobytes() == bcc2.tobytes()
    assert {k: v for k, v in stats.items() if k != "run_ms"} == {k: v for k, v in stats2.items() if k != "run_ms"}
    assert np.array_equal(cc.bridges(n, f, t), bridge)
    assert np.array_equal(cc.biconnected_components(n, f, t), bcc)
    assert stats["bridges"] == int(bridge.sum())
    assert stats["components"] == (int(bcc.max()) + 1 if len(bcc) else 0)
    assert stats["edges_inspected"] == 4 * len(f)  # forest and low / high passes each read every entry once
    loops = f == t
    touched = np.unique(np.concatenate([f[~loops], t[~loops]])) if len(f) else np.zeros(0)
    if n:
        from test_wcc_oracle import oracle_wcc
        comp = oracle_wcc(n, f, t)
        assert stats["trees"] == len(np.unique(comp[touched.astype(np.int64)]))
    return stats


def test_small_sizes(cc):
    rng = np.random.default_rng(1)
    for n in range(0, 34):
        for m in (0, n // 2, n, 2 * n, 4 * n):
            check(cc, n, rng.integers(0, max(n, 1), m), rng.integers(0, max(n, 1), m))


def test_trees_cycles_cliques(cc):
    rng = np.random.default_rng(2)
    n = 5000
    parent = np.array([rng.integers(0, v) for v in range(1, n)])  # random recursive tree
    stats = check(cc, n, parent, np.arange(1, n))
    assert stats["bridges"] == n - 1 and stats["components"] == n - 1
    v = rng.permutation(n)
    stats = check(cc, n, v, np.roll(v, 1))  # one cycle
    assert stats["bridges"] == 0 and stats["components"] == 1
    k = 60
    a, b = np.triu_indices(k, 1)
    stats = check(cc, k, a, b)
    assert stats["components"] == 1 and stats["forest_depth"] == 1
    blocks = [np.arange(i * 10, i * 10 + 10) for i in range(20)]  # 20 10-cycles chained through shared vertices
    f = np.concatenate([c for c in blocks] + [np.array([blocks[i][5] for i in range(19)])])
    t = np.concatenate([np.roll(c, 1) for c in blocks] + [np.array([blocks[i + 1][0] for i in range(19)])])
    stats = check(cc, 200, f, t)
    assert stats["bridges"] == 19 and stats["components"] == 39


def test_double_edges_and_self_loops(cc):
    rng = np.random.default_rng(3)
    n = 3000
    parent = np.array([rng.integers(max(0, v - 5), v) for v in range(1, n)])
    child = np.arange(1, n)
    doubled = rng.random(n - 1) < 0.3
    f = np.concatenate([parent, child[doubled], np.arange(0, n, 7)])  # some tree edges doubled (reversed), self-loops
    t = np.concatenate([child, parent[doubled], np.arange(0, n, 7)])
    stats = check(cc, n, f, t)
    assert stats["bridges"] == int((~doubled).sum())
    bcc = cc.biconnected_components(n, f, t)
    assert (bcc[len(f) - len(range(0, n, 7)):] == -1).all()
    check(cc, 4, [0, 0, 1, 2, 2, 3], [1, 1, 2, 2, 3, 3])


def test_long_paths_in_shuffled_id_order(cc):
    n = 100_000
    perm = np.random.default_rng(4).permutation(n)
    stats = check(cc, n, perm[:-1], perm[1:])
    assert stats["bridges"] == n - 1 and stats["forest_depth"] >= n // 2 - 1
    check(cc, n, perm[1:], perm[:-1])


def test_stars(cc):
    n = 300_000  # the hub's list crosses the one-block-per-vertex threshold
    leaves = np.arange(1, n)
    hub = np.zeros(n - 1, dtype=np.int64)
    check(cc, n, leaves, hub)
    check(cc, n, hub, leaves)
    check(cc, n, np.concatenate([hub, leaves[:999]]), np.concatenate([leaves, leaves[1:1000]]))  # leaves 1..1000 a fan
    hub = np.full(n // 2, n - 1)  # the hub is the largest id
    check(cc, n, hub, np.arange(n // 2))


def test_many_small_components(cc):
    n = 1_000_000
    rng = np.random.default_rng(5)
    stats = check(cc, n, rng.integers(0, n, n // 3), rng.integers(0, n, n // 3))
    assert stats["trees"] > 100_000


@pytest.mark.parametrize("n,m", [(5000, 2500), (5000, 5000), (5000, 20000), (200_000, 150_000), (200_000, 300_000),
                                 (200_000, 800_000)])
def test_erdos_renyi(cc, n, m):
    rng = np.random.default_rng(n + m)
    check(cc, n, rng.integers(0, n, m), rng.integers(0, n, m))


@pytest.mark.parametrize("scale", [20, 22])
def test_rmat(cc, scale):
    n = 1 << scale
    f, t = oracle_rmat_edges(scale)
    stats = check(cc, n, f, t)
    assert stats["bridges"] > 0 and stats["components"] > 1


def test_argument_errors(cc):
    import ctypes
    from memgraph_b200 import _native as N
    lib = N.lib()
    s = np.array([0, 1], dtype=np.uint64)
    t = s + 1
    assert lib.mgb200_bridges(3, 2, s.ctypes.data, t.ctypes.data, None) == N.ERR_INVALID_ARGUMENT
    assert lib.mgb200_biconnected_components(3, 2, s.ctypes.data, t.ctypes.data, None) == N.ERR_INVALID_ARGUMENT
    assert lib.mgb200_biconnectivity_run(None, 0, None, None, None, None, None) == N.ERR_INVALID_ARGUMENT
    assert lib.mgb200_bridges(0, 0, None, None, None) == N.OK
    assert lib.mgb200_biconnected_components(0, 0, None, None, None) == N.OK
    with cc.BfsGraph(3, s, t) as g:
        assert lib.mgb200_biconnectivity_run(g._h, 1, s.ctypes.data, t.ctypes.data, None, None, None) == \
            N.ERR_INVALID_ARGUMENT  # m differs from the graph's
        assert lib.mgb200_biconnectivity_run(g._h, 2, None, None, None, None, None) == N.ERR_INVALID_ARGUMENT
        bad = np.array([0, 3], dtype=np.uint64)
        assert lib.mgb200_biconnectivity_run(g._h, 2, s.ctypes.data, bad.ctypes.data, None, None, None) == \
            N.ERR_INVALID_ARGUMENT  # endpoint out of range
        assert lib.mgb200_biconnectivity_run(g._h, 2, s.ctypes.data, t.ctypes.data, None, None, None) == N.OK
        out = np.zeros(2, dtype=np.int64)
        assert lib.mgb200_biconnectivity_run(g._h, 2, s.ctypes.data, t.ctypes.data, None, out.ctypes.data, None) == N.OK
        assert out.tolist() == [0, 1]
    st = N.BiconnectivityStats()
    with cc.BfsGraph(0, [], []) as g:
        assert lib.mgb200_biconnectivity_run(g._h, 0, None, None, None, None, ctypes.byref(st)) == N.OK
        assert st.components == 0 and st.kernel_launches == 0

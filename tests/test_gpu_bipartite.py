"""Maximum bipartite matching on the device (memgraph_b200/csrc/bipartite_matching.cu) against oracle/bipartite_oracle.c,
which tests/test_bipartite_oracle.py pins to the reference.  Every run is also checked by its own certificate: the
pairs form a matching of graph edges, and the returned cover covers every edge with as many vertices as there are
pairs, which proves the matching maximum (Konig's theorem) where no oracle is quick."""
import numpy as np
import pytest

from test_bipartite_oracle import bipartite_rmat, e2e_cases, golden, oracle_matching, seeded_graphs, split, unit_cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mm():
    from memgraph_b200 import matching
    return matching


def certify(n, f, t, mate, cover, stats):
    """The pairs are a matching of edges, the cover covers every edge, and both have stats["matched"] elements."""
    matched = stats["matched"]
    if not stats["bipartite"]:
        assert matched == 0 and (mate == -1).all() and not cover.any()
        return
    v = np.flatnonzero(mate >= 0)
    assert (mate[mate[v]] == v).all() and len(v) == 2 * matched
    keys = np.unique(np.minimum(f, t) * np.uint64(n) + np.maximum(f, t))
    a = v[v < mate[v]].astype(np.uint64)
    assert np.isin(a * np.uint64(n) + mate[a].astype(np.uint64), keys).all()
    assert (cover[f] | cover[t]).all() and int(cover.sum()) == matched
    assert stats["initial_matched"] <= matched and (stats["phases"] >= 1) == (n > 0)


def check(mm, n, f, t, oracle=True):
    """Resident run (twice: byte-identical, stats included), one-shot call, certificate and, unless told otherwise,
    the oracle.  -> stats."""
    f = np.asarray(f, dtype=np.uint64)
    t = np.asarray(t, dtype=np.uint64)
    with mm.BfsGraph(n, f, t) as g:
        mate, cover, stats = mm.bipartite_matching_run(g)
        mate2, cover2, stats2 = mm.bipartite_matching_run(g)
    assert mate.tobytes() == mate2.tobytes() and cover.tobytes() == cover2.tobytes()
    assert {k: x for k, x in stats.items() if k != "run_ms"} == {k: x for k, x in stats2.items() if k != "run_ms"}
    certify(n, f, t, mate, cover, stats)
    assert mm.maximum_bipartite_matching(n, f, t) == stats["matched"]
    if oracle:
        assert stats["matched"] == oracle_matching(n, f, t)
    return stats


def test_fixtures(mm):
    for name, n, edges, expected in list(e2e_cases()) + list(unit_cases()):
        assert check(mm, n, *split(edges))["matched"] == expected, name
    for (name, n, f, t), rec in zip(seeded_graphs(), golden()["seeded"]):
        assert check(mm, n, f, t)["matched"] == rec["expected"], name


def test_random_small_graphs(mm):
    rng = np.random.default_rng(11)
    for _ in range(300):
        n = int(rng.integers(1, 40))
        m = int(rng.integers(0, 3 * n))
        f, t = rng.integers(0, n, m), rng.integers(0, n, m)
        if rng.random() < 0.7:
            side = rng.integers(0, 2, n)
            keep = side[f] != side[t]
            f, t = f[keep], t[keep]
        check(mm, n, f, t)


def test_either_orientation(mm):
    rng = np.random.default_rng(12)
    a, b, m = 3000, 2000, 9000
    f, t = rng.integers(0, a, m), a + rng.integers(0, b, m)
    flip = rng.random(m) < 0.5
    forward = check(mm, a + b, f, t)
    assert check(mm, a + b, t, f)["matched"] == forward["matched"]
    assert check(mm, a + b, np.where(flip, t, f), np.where(flip, f, t))["matched"] == forward["matched"]


def test_odd_component_makes_it_zero(mm):
    rng = np.random.default_rng(13)
    f, t = rng.integers(0, 500, 2000), 500 + rng.integers(0, 500, 2000)
    assert check(mm, 1005, f, t)["matched"] > 0
    cycle = 1000 + np.arange(5)  # a 5-cycle in a component of its own
    stats = check(mm, 1005, np.concatenate([f, cycle]), np.concatenate([t, np.roll(cycle, 1)]))
    assert stats["bipartite"] == 0 and stats["matched"] == 0


@pytest.mark.parametrize("a,b", [(1, 1), (1, 7), (7, 1), (13, 40), (200, 150)])
def test_complete_bipartite(mm, a, b):
    f, t = np.repeat(np.arange(a), b), a + np.tile(np.arange(b), a)
    assert check(mm, a + b, f, t)["matched"] == min(a, b)


@pytest.mark.parametrize("degree", [16, 17, 4096, 4097])
def test_stars(mm, degree):
    """The hub's list on each side of the thread / warp / block walk thresholds, the hub on the left (id 0, the root)
    and on the right (the largest id, one level below leaf 0)."""
    leaves = np.arange(1, degree + 1)
    stats = check(mm, degree + 1, np.zeros(degree), leaves)
    assert stats["matched"] == 1 and stats["left_vertices"] == 1
    n = degree + 1
    stats = check(mm, n, np.full(degree, n - 1), np.arange(degree))
    assert stats["matched"] == 1 and stats["left_vertices"] == degree
    # two hubs sharing their leaves: still one pair per hub
    f = np.concatenate([np.zeros(degree), np.full(degree, degree + 1)])
    t = np.concatenate([leaves, leaves])
    assert check(mm, degree + 2, f, t)["matched"] == 2


def test_long_path_and_even_cycle_in_shuffled_order(mm):
    n = 20_000
    perm = np.random.default_rng(14).permutation(n)
    stats = check(mm, n, perm[:-1], perm[1:])
    assert stats["matched"] == n // 2
    stats = check(mm, n, perm, np.roll(perm, -1))  # even cycle
    assert stats["matched"] == n // 2
    odd = perm[:-1]
    assert check(mm, n, odd, np.roll(odd, -1))["bipartite"] == 0  # odd cycle


@pytest.mark.parametrize("scale", [16, 18, 20])
def test_bipartite_rmat(mm, scale):
    n, f, t = bipartite_rmat(scale)
    stats = check(mm, n, f, t)
    assert stats["bipartite"] == 1 and stats["matched"] > stats["initial_matched"] > 0


def test_bipartite_rmat_22_by_certificate(mm):
    n, f, t = bipartite_rmat(22)
    stats = check(mm, n, f, t, oracle=False)
    assert stats["bipartite"] == 1 and stats["matched"] > 0


def test_should_abort(mm):
    from memgraph_b200 import MgB200Error
    rng = np.random.default_rng(15)
    f, t = rng.integers(0, 1000, 4000), 1000 + rng.integers(0, 1000, 4000)
    calls = []
    with mm.BfsGraph(2000, f, t) as g:
        with pytest.raises(MgB200Error, match="aborted"):
            mm.bipartite_matching_run(g, should_abort=lambda: calls.append(1) or True)
        assert calls == [1]  # polled before the first phase
        mate, cover, stats = mm.bipartite_matching_run(g, should_abort=lambda: False)
    certify(2000, f.astype(np.uint64), t.astype(np.uint64), mate, cover, stats)


def test_empty_graphs(mm):
    with mm.BfsGraph(0, [], []) as g:
        mate, cover, stats = mm.bipartite_matching_run(g)
    assert len(mate) == 0 and len(cover) == 0
    assert stats["bipartite"] == 1 and stats["matched"] == 0 and stats["kernel_launches"] == 0
    assert mm.maximum_bipartite_matching(0, [], []) == 0
    stats = check(mm, 50, [], [])
    assert stats["matched"] == 0 and stats["left_vertices"] == 50 and stats["phases"] == 1

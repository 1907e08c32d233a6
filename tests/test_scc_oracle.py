"""oracle/scc_oracle.c -- the iterative Tarjan behind the strongly-connected-components tests -- against networkx's
partitions recorded in tests/golden/scc_cases.json (the reference's nxalg.strongly_connected_components runs networkx on
the MultiDiGraph of all vertices and edges), against networkx and scipy live where they are installed, and against a
brute-force transitive closure on small graphs."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

from _checkers import oracle_rmat_edges

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
SCC_ORACLE_SRC = os.path.join(REPO, "oracle", "scc_oracle.c")
SCC_ORACLE_SO = os.path.join(REPO, "oracle", "_build", "libscc_oracle.so")
_oracle = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        if not os.path.exists(SCC_ORACLE_SO) or os.path.getmtime(SCC_ORACLE_SO) < os.path.getmtime(SCC_ORACLE_SRC):
            subprocess.run(["make", "-s", "-C", os.path.join(REPO, "oracle"), "-f", "scc.mk", "oracle"], check=True)
        L = ctypes.CDLL(SCC_ORACLE_SO)
        L.oracle_scc.argtypes = [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        _oracle = L
    return _oracle


def oracle_scc(n, frm, to):
    """Strongly connected component of every vertex (int64[n]), numbered in the order of each one's smallest id."""
    frm = np.ascontiguousarray(frm, dtype=np.uint64)
    to = np.ascontiguousarray(to, dtype=np.uint64)
    out = np.zeros(int(n), dtype=np.int64)
    rc = oracle_lib().oracle_scc(int(n), len(frm), frm.ctypes.data, to.ctypes.data, out.ctypes.data)
    assert rc == 0, rc
    return out


def canonical(labels):
    """Any labelling of a partition -> the numbering by each part's smallest member."""
    labels = np.asarray(labels)
    _, first, inverse = np.unique(labels, return_index=True, return_inverse=True)
    rank = np.empty(len(first), dtype=np.int64)
    rank[np.argsort(first, kind="stable")] = np.arange(len(first))
    return rank[inverse.reshape(-1)]


def handmade_graphs():
    """(name, n, edges) with the shapes that decide a partition: cycles, self-loops, multi-edges, chains of blocks."""
    out = [("empty", 0, []), ("one_vertex", 1, []), ("self_loop", 1, [(0, 0)]), ("two_isolated", 2, []),
           ("one_edge", 2, [(0, 1)]), ("two_cycle", 2, [(0, 1), (1, 0)]),
           ("doubled_edge", 3, [(0, 1), (0, 1), (1, 2)]),
           ("triangle_and_tail", 5, [(0, 1), (1, 2), (2, 0), (2, 3), (3, 4)]),
           ("tail_into_cycle", 5, [(4, 3), (3, 0), (0, 1), (1, 2), (2, 0)]),
           ("two_cycles_bridged", 6, [(0, 1), (1, 0), (1, 2), (2, 3), (3, 4), (4, 2), (5, 5)]),
           ("figure_eight", 5, [(0, 1), (1, 2), (2, 0), (2, 3), (3, 4), (4, 2)]),
           ("reverse_ids", 4, [(3, 2), (2, 1), (1, 3), (0, 3)]),
           ("dag", 6, [(5, 4), (5, 3), (4, 2), (3, 2), (2, 1), (1, 0)])]
    # the textbook example (Cormen et al., figure 22.9) with shuffled ids
    ids = [6, 2, 7, 0, 3, 5, 1, 4]
    book = [(0, 1), (1, 2), (1, 4), (1, 5), (2, 3), (2, 6), (3, 2), (3, 7), (4, 0), (4, 5), (5, 6), (6, 5), (6, 7),
            (7, 7)]
    out.append(("cormen_22_9", 8, [(ids[a], ids[b]) for a, b in book]))
    return out


def block_chain(blocks, size, rng, ascending):
    """`blocks` cycles of `size` vertices, each with one edge into the next; ids shuffled, or ascending along the
    chain.  -> (n, from, to)."""
    n = blocks * size
    f, t = [], []
    for b in range(blocks):
        base = b * size
        for i in range(size):
            f.append(base + i)
            t.append(base + (i + 1) % size)
        if b + 1 < blocks:
            f.append(base)
            t.append(base + size)
    perm = np.arange(n) if ascending else rng.permutation(n)
    return n, perm[np.array(f, dtype=np.int64)], perm[np.array(t, dtype=np.int64)]


def seeded_graphs():
    """(name, n, from, to): random directed multigraphs with self-loops at several densities, and chains of blocks."""
    rng = np.random.default_rng(20261019)
    out = []
    for n, m in [(40, 30), (100, 120), (300, 400), (500, 1000), (800, 960), (1000, 4000)]:
        out.append((f"random_{n}_{m}", n, rng.integers(0, n, m), rng.integers(0, n, m)))
    out.append(("block_chain_shuffled", *block_chain(60, 5, rng, False)))
    out.append(("block_chain_ascending", *block_chain(40, 3, rng, True)))
    return out


def golden():
    return json.load(open(os.path.join(GOLDEN, "scc_cases.json")))


def brute_force(n, f, t):
    """Components from the transitive closure: u and v share one iff each reaches the other."""
    reach = np.eye(n, dtype=bool)
    reach[np.asarray(f, dtype=np.int64), np.asarray(t, dtype=np.int64)] = True
    for k in range(n):
        reach |= reach[:, k:k + 1] & reach[k:k + 1, :]
    both = reach & reach.T
    return np.array([np.flatnonzero(both[v])[0] for v in range(n)], dtype=np.int64)  # smallest member


def test_golden_cases():
    spec = golden()
    hand = handmade_graphs()
    assert [c["name"] for c in spec["handmade"]] == [name for name, _, _ in hand]
    for (name, n, edges), case in zip(hand, spec["handmade"]):
        e = np.array(edges, dtype=np.int64).reshape(-1, 2)
        assert oracle_scc(n, e[:, 0], e[:, 1]).tolist() == case["components"], name
    seeded = seeded_graphs()
    assert [c["name"] for c in spec["seeded"]] == [name for name, *_ in seeded]
    for (name, n, f, t), case in zip(seeded, spec["seeded"]):
        assert oracle_scc(n, f, t).tolist() == case["components"], name


def test_against_networkx_and_scipy():
    nx = pytest.importorskip("networkx")
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    rng = np.random.default_rng(11)
    for n, m in [(1, 0), (2, 2), (30, 25), (200, 200), (200, 260), (1000, 1200), (1000, 2000), (3000, 12000)]:
        f, t = rng.integers(0, n, m), rng.integers(0, n, m)
        got = oracle_scc(n, f, t)
        g = nx.MultiDiGraph()
        g.add_nodes_from(range(n))
        g.add_edges_from(zip(f.tolist(), t.tolist()))
        labels = np.empty(n, dtype=np.int64)
        for i, comp in enumerate(nx.strongly_connected_components(g)):
            labels[list(comp)] = i
        assert np.array_equal(got, canonical(labels)), (n, m)
        _, lab = connected_components(coo_matrix((np.ones(m), (f, t)), shape=(n, n)), directed=True,
                                      connection="strong")
        assert np.array_equal(got, canonical(lab)), (n, m)


def test_against_the_transitive_closure():
    rng = np.random.default_rng(12)
    for n, m in [(1, 1), (3, 4), (8, 10), (20, 25), (40, 50), (60, 120)]:
        for _ in range(5):
            f, t = rng.integers(0, n, m), rng.integers(0, n, m)
            assert np.array_equal(oracle_scc(n, f, t), canonical(brute_force(n, f, t))), (n, m)
    for name, n, edges in handmade_graphs():
        e = np.array(edges, dtype=np.int64).reshape(-1, 2)
        assert np.array_equal(oracle_scc(n, e[:, 0], e[:, 1]), canonical(brute_force(n, e[:, 0], e[:, 1]))), name


def test_rmat_16_against_scipy():
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    n = 1 << 16
    f, t = oracle_rmat_edges(16)
    got = oracle_scc(n, f, t)
    _, lab = connected_components(coo_matrix((np.ones(len(f)), (f.astype(np.int64), t.astype(np.int64))),
                                             shape=(n, n)), directed=True, connection="strong")
    assert np.array_equal(got, canonical(lab))
    sizes = np.bincount(got)
    assert sizes.max() > n // 3 and (sizes[sizes != sizes.max()] == 1).all()  # one giant, the rest singletons


def test_long_cycle_does_not_recurse():
    n = 2_000_000
    perm = np.random.default_rng(13).permutation(n)
    got = oracle_scc(n, perm, np.roll(perm, -1))
    assert not got.any()
    got = oracle_scc(n, perm[:-1], perm[1:])
    assert np.array_equal(got, np.arange(n))


def test_numbering_and_errors():
    rng = np.random.default_rng(14)
    f, t = rng.integers(0, 500, 600), rng.integers(0, 500, 600)
    comp = oracle_scc(500, f, t)
    first = np.unique(comp, return_index=True)[1]
    assert np.array_equal(comp[np.sort(first)], np.arange(len(first)))  # numbers appear in vertex order
    with pytest.raises(AssertionError):
        oracle_scc(3, [0, 3], [1, 2])  # endpoint out of range
    assert len(oracle_scc(0, [], [])) == 0

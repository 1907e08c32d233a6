"""oracle/bipartite_oracle.c -- the plain-C restatement of the reference's maximum bipartite matching (colouring, then
Hopcroft-Karp) -- against the reference's e2e fixtures and gtest cases, the reference module's recorded answers on the
seeded graphs below (tests/golden/bipartite_cases.json), brute force on small multigraphs, scipy on larger bipartite
graphs and, where oracle/_ref was built, the live reference module."""
import ctypes
import functools
import json
import os
import subprocess

import numpy as np

from _bc_host import isolated
from _checkers import oracle_rmat_edges

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
ORACLE_SRC = os.path.join(REPO, "oracle", "bipartite_oracle.c")
ORACLE_SO = os.path.join(REPO, "oracle", "_build", "libbipartite_oracle.so")
REF_MODULE_SO = os.path.join(REPO, "oracle", "_ref", "bipartite_matching_reference.so")
_oracle = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        if not os.path.exists(ORACLE_SO) or os.path.getmtime(ORACLE_SO) < os.path.getmtime(ORACLE_SRC):
            subprocess.run(["make", "-s", "-C", os.path.join(REPO, "oracle"), "-f", "bipartite.mk", "oracle"],
                           check=True)
        L = ctypes.CDLL(ORACLE_SO)
        L.oracle_bipartite_matching.argtypes = [ctypes.c_uint64, ctypes.c_uint64] + [ctypes.c_void_p] * 4
        _oracle = L
    return _oracle


def oracle_matching(n, frm, to, with_mate=False):
    """The reference's answer: 0 with a self-loop or an odd cycle, else the size of a maximum matching.  with_mate:
    -> (answer, int64[n] partners, -1 where unmatched)."""
    frm = np.ascontiguousarray(frm, dtype=np.uint64)
    to = np.ascontiguousarray(to, dtype=np.uint64)
    out = ctypes.c_uint64(0)
    mate = np.full(int(n), -1, dtype=np.int64)
    rc = oracle_lib().oracle_bipartite_matching(int(n), len(frm), frm.ctypes.data, to.ctypes.data, ctypes.byref(out),
                                                mate.ctypes.data if with_mate and n else None)
    assert rc == 0, rc
    return (int(out.value), mate) if with_mate else int(out.value)


def bipartite_rmat(scale, seed=42):
    """RMAT(scale, 16 * 2^scale edges) as a bipartite graph: (u, v) -> (u, 2^scale + v), 2 * 2^scale vertices."""
    f, t = oracle_rmat_edges(scale, seed=seed)
    return 2 << scale, f, t + (1 << scale)


def seeded_graphs():
    """(name, n, from, to) whose answers tests/golden/bipartite_cases.json records from the reference module: random
    bipartite multigraphs with isolated vertices, the same with one odd cycle or one self-loop added, random
    non-bipartite graphs, and bipartite RMAT at scales 10 and 12."""
    rng = np.random.default_rng(20261018)
    out = []
    for name, a, b, m in [("bip_sparse", 60, 80, 70), ("bip_medium", 300, 200, 600), ("bip_dense", 150, 150, 3000),
                          ("bip_unbalanced", 40, 700, 900)]:
        f, t = rng.integers(0, a, m), a + rng.integers(0, b, m)
        f, t = np.concatenate([f, f[:7]]), np.concatenate([t, t[:7]])  # multi-edges for certain
        out.append((name, a + b + 5, f, t))  # 5 isolated vertices at the end
    f, t = rng.integers(0, 100, 300), 100 + rng.integers(0, 100, 300)
    out.append(("bip_plus_triangle", 203, np.concatenate([f, [200, 201, 202]]), np.concatenate([t, [201, 202, 200]])))
    out.append(("bip_plus_self_loop", 200, np.concatenate([f, [150]]), np.concatenate([t, [150]])))
    out.append(("bip_reversed_edges", 200, t, f))
    for name, n, m in [("random_sparse", 400, 150), ("random_dense", 300, 1200)]:
        out.append((name, n, rng.integers(0, n, m), rng.integers(0, n, m)))
    for scale in (10, 12):
        out.append((f"bip_rmat{scale}",) + bipartite_rmat(scale))
    return out


def golden():
    return json.load(open(os.path.join(GOLDEN, "bipartite_cases.json")))


def e2e_cases():
    """(name, n, dense edges, expected): nodes in creation order."""
    for case in golden()["e2e"]:
        dense = {v: i for i, v in enumerate(case["nodes"])}
        yield case["name"], len(dense), [(dense[a], dense[b]) for a, b in case["edges"]], case["expected"]


def unit_cases():
    """(name, n, edges, expected) of the gtest file; a case without a stated count has the reference module's."""
    for case in golden()["unit"]:
        yield case["name"], case["n"], case["edges"], case["expected"]


def split(edges):
    e = np.array(edges, dtype=np.int64).reshape(-1, 2)
    return e[:, 0], e[:, 1]


def brute_force(n, edges):
    """Bipartite by trying every 2-colouring, then a maximum matching by memoised search over vertex subsets."""
    if any(a == b for a, b in edges):
        return 0
    if edges:
        e = np.array(edges)
        colours = (np.arange(1 << n)[:, None] >> np.arange(n)[None, :]) & 1
        if not (colours[:, e[:, 0]] != colours[:, e[:, 1]]).all(axis=1).any():
            return 0
    adj = [0] * n
    for a, b in edges:
        adj[a] |= 1 << b
        adj[b] |= 1 << a

    @functools.lru_cache(maxsize=None)
    def best(mask):
        if mask == 0:
            return 0
        v = (mask & -mask).bit_length() - 1
        rest = mask & ~(1 << v)
        r = best(rest)
        cand = adj[v] & rest
        while cand:
            w = (cand & -cand).bit_length() - 1
            cand &= cand - 1
            r = max(r, 1 + best(rest & ~(1 << w)))
        return r

    return best((1 << n) - 1)


def test_e2e_fixtures():
    cases = list(e2e_cases())
    assert sorted(name for name, *_ in cases) == ["test_chain", "test_cycle", "test_empty", "test_hierarchy"]
    for name, n, edges, expected in cases:
        assert oracle_matching(n, *split(edges)) == expected, name


def test_gtest_cases():
    cases = list(unit_cases())
    assert len(cases) == 16
    for name, n, edges, expected in cases:
        assert oracle_matching(n, *split(edges)) == expected, name


def test_recorded_reference_answers():
    recorded = golden()["seeded"]
    graphs = seeded_graphs()
    assert [c["name"] for c in recorded] == [name for name, *_ in graphs]
    for (name, n, f, t), call in zip(graphs, recorded):
        assert (n, len(f)) == (call["n"], call["m"]), name
        assert oracle_matching(n, f, t) == call["expected"], name
    assert any(c["expected"] == 0 for c in recorded) and all(c["expected"] > 0 for c in recorded[:4])


def test_brute_force_small_multigraphs():
    rng = np.random.default_rng(7)
    zero = 0
    for _ in range(3000):
        n = int(rng.integers(1, 10))
        m = int(rng.integers(0, 2 * n + 1))
        edges = [(int(a), int(b)) for a, b in zip(rng.integers(0, n, m), rng.integers(0, n, m))]
        if rng.random() < 0.5:  # keep half of them bipartite: drop the edges inside a random side
            side = rng.integers(0, 2, n)
            edges = [(a, b) for a, b in edges if side[a] != side[b]]
        if edges and rng.random() < 0.2:
            edges += edges[: int(rng.integers(1, len(edges) + 1))]  # duplicates
        f, t = split(edges)
        got, mate = oracle_matching(n, f, t, with_mate=True)
        assert got == brute_force(n, edges), (n, edges)
        zero += got == 0 and bool(edges)
        pairs = {(int(v), int(mate[v])) for v in range(n) if mate[v] >= 0}
        assert len(pairs) == 2 * got and all((w, v) in pairs for v, w in pairs)
        assert all((a, b) in set(edges) or (b, a) in set(edges) for a, b in pairs)
    assert zero > 300  # odd cycles and self-loops were exercised


def test_scipy_random_bipartite():
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import maximum_bipartite_matching
    rng = np.random.default_rng(9)
    for a, b, m in [(1, 1, 1), (10, 3, 12), (500, 700, 900), (4000, 3000, 20000), (1 << 15, 1 << 15, 1 << 17),
                    (1 << 16, 1 << 14, 1 << 18)]:
        u, v = rng.integers(0, a, m), rng.integers(0, b, m)
        expected = int((maximum_bipartite_matching(csr_matrix((np.ones(m), (u, v)), shape=(a, b)),
                                                   perm_type="column") >= 0).sum())
        assert oracle_matching(a + b, u, a + v) == expected, (a, b, m)
        assert oracle_matching(a + b, a + v, u) == expected, (a, b, m)  # the other orientation


def test_argument_errors():
    out = ctypes.c_uint64(0)
    f = np.array([0, 3], dtype=np.uint64)
    assert oracle_lib().oracle_bipartite_matching(3, 2, f.ctypes.data, f.ctypes.data, ctypes.byref(out), None) == 1
    assert oracle_matching(0, [], []) == 0


@isolated
def test_live_reference_module():
    """The reference's own module through the host equals the oracle on the fixtures and on random graphs."""
    if not os.path.exists(REF_MODULE_SO):
        return  # oracle/_ref/bipartite_matching_reference.so is built only where a reference checkout exists
    import test_bipartite_module as bm
    rng = np.random.default_rng(33)
    graphs = [(name, n, *split(edges)) for name, n, edges, _ in list(e2e_cases()) + list(unit_cases())]
    for n, m in [(6, 5), (40, 30), (300, 200)]:
        side = rng.integers(0, 2, n)
        f, t = rng.integers(0, n, m), rng.integers(0, n, m)
        keep = side[f] != side[t]
        graphs += [("random", n, f, t), ("random_bipartite", n, f[keep], t[keep])]
    with bm.Module(REF_MODULE_SO) as ref:
        for name, n, f, t in graphs:
            assert bm.call(ref, n, f, t) == oracle_matching(n, f, t), name


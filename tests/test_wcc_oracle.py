"""oracle/wcc_oracle.c -- the plain-C restatement of the reference's weakly connected components -- against the
reference's e2e fixtures, the recorded rows of the reference's own module (sha256 in
tests/golden/wcc_ref_module_rows.json) and, where oracle/_ref was built, the live reference module on random graphs."""
import ctypes
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from _bc_host import isolated

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
WCC_ORACLE_SRC = os.path.join(REPO, "oracle", "wcc_oracle.c")
WCC_ORACLE_SO = os.path.join(REPO, "oracle", "_build", "libwcc_oracle.so")
_oracle = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        if not os.path.exists(WCC_ORACLE_SO) or os.path.getmtime(WCC_ORACLE_SO) < os.path.getmtime(WCC_ORACLE_SRC):
            subprocess.run(["make", "-s", "-C", os.path.join(REPO, "oracle"), "-f", "wcc.mk", "oracle"], check=True)
        L = ctypes.CDLL(WCC_ORACLE_SO)
        L.oracle_wcc.argtypes = [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        _oracle = L
    return _oracle


def oracle_wcc(n, frm, to):
    """Component number of every vertex (int64[n]), numbered in BFS order from the vertices in dense order."""
    frm = np.ascontiguousarray(frm, dtype=np.uint64)
    to = np.ascontiguousarray(to, dtype=np.uint64)
    out = np.zeros(int(n), dtype=np.int64)
    rc = oracle_lib().oracle_wcc(int(n), len(frm), frm.ctypes.data, to.ctypes.data, out.ctypes.data)
    assert rc == 0, rc
    return out


def rows_sha256(rows):
    return hashlib.sha256(np.ascontiguousarray(rows, dtype=np.int64).tobytes()).hexdigest()


def e2e_steps():
    """(case name, node ids in creation order = dense order, edges as dense pairs, expected rows) per query step."""
    for case in json.load(open(os.path.join(GOLDEN, "wcc_e2e_cases.json")))["cases"]:
        for step in case["steps"]:
            dense = {v: i for i, v in enumerate(step["nodes"])}
            edges = [(dense[a], dense[b]) for a, b in step["edges"]]
            yield case["name"], step["nodes"], edges, [(o["node_id"], o["component_id"]) for o in step["output"]]


def test_e2e_fixtures():
    spec = json.load(open(os.path.join(GOLDEN, "wcc_e2e_cases.json")))
    assert len(spec["cases"]) == 5
    steps = list(e2e_steps())
    assert len(steps) == 9  # the two online cases: one graph per query step
    for name, nodes, edges, expected in steps:
        e = np.array(edges, dtype=np.int64).reshape(-1, 2)
        comp = oracle_wcc(len(nodes), e[:, 0], e[:, 1])
        assert sorted(zip(nodes, comp.tolist())) == expected, name


def test_numbering_follows_the_smallest_vertex():
    rng = np.random.default_rng(8)
    for n, m in [(1, 0), (2, 1), (50, 20), (400, 300), (3000, 2000)]:
        f, t = rng.integers(0, n, m), rng.integers(0, n, m)
        comp = oracle_wcc(n, f, t)
        first = np.unique(comp, return_index=True)[1]
        assert np.array_equal(comp[np.sort(first)], np.arange(len(first)))  # numbers appear in vertex order
        assert (comp[f] == comp[t]).all()
        # the same partition as scipy's
        from scipy.sparse import coo_matrix
        from scipy.sparse.csgraph import connected_components
        k, labels = connected_components(coo_matrix((np.ones(m), (f, t)), shape=(n, n)), directed=True,
                                         connection="weak")
        assert k == len(first)
        assert len({(a, b) for a, b in zip(labels.tolist(), comp.tolist())}) == k
    with pytest.raises(AssertionError):
        oracle_wcc(3, [0, 3], [1, 2])  # endpoint out of range
    assert len(oracle_wcc(0, [], [])) == 0


def test_matches_the_recorded_reference_module_rows():
    """The reference module's rows, recorded as sha256 of the (gid, component) rows sorted by gid, are the oracle's on
    the module's graph view (vertices in ascending gid order)."""
    import test_wcc_module as wm
    recorded = wm.recorded_rows()["graphs"]
    assert [c["name"] for c in recorded] == [name for name, *_ in wm.wcc_scattered_graphs()]
    for (name, gids, src, dst), call in zip(wm.wcc_scattered_graphs(), recorded):
        rows = wm.module_oracle(gids, src, dst)
        assert rows_sha256(rows) == call["rows_sha256"], name
        assert len(rows) == call["rows"] and int(rows[:, 1].max()) + 1 == call["components"], name


@isolated
def test_live_reference_module():
    """The reference's own module through the host: its rows (a gid -> component mapping) equal the oracle's on random
    scattered-gid graphs, transactional and analytical with hidden vertices, and on the e2e fixtures."""
    import test_wcc_module as wm
    if not wm.HAVE_REF_MODULE:
        return  # oracle/_ref/weakly_connected_components_reference.so is built only where a reference checkout exists
    rng = np.random.default_rng(31)
    with wm.Module(wm.REF_WCC_MODULE_SO) as ref:
        wm.check_e2e_fixtures(ref)
        for name, gids, src, dst in wm.wcc_scattered_graphs():
            with wm.Graph(gids, src, dst) as g:
                assert np.array_equal(wm.rows_of(*ref.call(g)), wm.module_oracle(gids, src, dst)), name
        for n, m in [(5, 3), (64, 40), (700, 500), (2000, 2600)]:
            gids = rng.choice(np.arange(20 * n, dtype=np.int64), size=n, replace=False)
            src, dst = gids[rng.integers(0, n, m)], gids[rng.integers(0, n, m)]
            with wm.Graph(gids, src, dst) as g:
                assert np.array_equal(wm.rows_of(*ref.call(g)), wm.module_oracle(gids, src, dst)), (n, m)
            hidden = rng.choice(gids, size=max(1, n // 10), replace=False)
            with wm.Graph(gids, src, dst, transactional=False) as g:
                for gid in hidden:
                    g.hide_vertex(int(gid))
                assert np.array_equal(wm.rows_of(*ref.call(g)), wm.module_oracle(gids, src, dst, hidden)), (n, m)

"""oracle/biconnectivity_oracle.c -- the iterative Hopcroft-Tarjan restatement of the reference's bridges and
biconnected components -- against the recorded rows of the reference's own modules
(tests/golden/biconnectivity_ref_module_rows.json), the handmade graphs of the reference's unit tests, the e2e fixtures,
the brute-force definitions on small random multigraphs and, where oracle/_ref was built, the live reference modules."""
import ctypes
import json
import os
import subprocess
from collections import defaultdict

import numpy as np
import pytest

from _bc_host import isolated

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
ORACLE_SRC = os.path.join(REPO, "oracle", "biconnectivity_oracle.c")
ORACLE_SO = os.path.join(REPO, "oracle", "_build", "libbiconnectivity_oracle.so")
_oracle = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        if not os.path.exists(ORACLE_SO) or os.path.getmtime(ORACLE_SO) < os.path.getmtime(ORACLE_SRC):
            subprocess.run(["make", "-s", "-C", os.path.join(REPO, "oracle"), "-f", "biconnectivity.mk", "oracle"],
                           check=True)
        L = ctypes.CDLL(ORACLE_SO)
        L.oracle_biconnectivity.argtypes = [ctypes.c_uint64, ctypes.c_uint64] + [ctypes.c_void_p] * 4
        _oracle = L
    return _oracle


def oracle_biconnectivity(n, frm, to):
    """-> (uint8[m] bridge flags, int64[m] components numbered by first edge, -1 for self-loops)."""
    frm = np.ascontiguousarray(frm, dtype=np.uint64)
    to = np.ascontiguousarray(to, dtype=np.uint64)
    bridge, bcc = np.zeros(len(frm), dtype=np.uint8), np.zeros(len(frm), dtype=np.int64)
    rc = oracle_lib().oracle_biconnectivity(int(n), len(frm), frm.ctypes.data, to.ctypes.data, bridge.ctypes.data,
                                            bcc.ctypes.data)
    assert rc == 0, rc
    return bridge, bcc


def bcc_partition(rows):
    """Rows (component, a, b) -> the partition of the distinct unordered non-loop pairs {a, b} into components."""
    groups, seen = defaultdict(set), {}
    for c, a, b in rows:
        a, b = int(a), int(b)
        if a == b:
            continue
        pair = (min(a, b), max(a, b))
        assert seen.setdefault(pair, int(c)) == int(c), f"{pair} is in two components"
        groups[int(c)].add(pair)
    return {frozenset(g) for g in groups.values()}


def first_edge_numbering(keys):
    """Relabel arbitrary per-edge keys (None = no component) by the order of each key's first edge."""
    out, number = np.full(len(keys), -1, dtype=np.int64), {}
    for e, k in enumerate(keys):
        if k is not None:
            out[e] = number.setdefault(k, len(number))
    return out


def _components(n, edges):
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b in edges:
        parent[find(a)] = find(b)
    return [find(x) for x in range(n)]


def brute_force(n, f, t):
    """The definitions: e is a bridge iff deleting it separates its endpoints; two non-loop edges share a component iff
    they are connected and no single vertex deletion separates their remaining endpoints."""
    m = len(f)
    edges = [(int(a), int(b)) for a, b in zip(f, t)]
    bridge = np.zeros(m, dtype=np.uint8)
    for e, (a, b) in enumerate(edges):
        if a != b:
            comp = _components(n, edges[:e] + edges[e + 1:])
            bridge[e] = comp[a] != comp[b]
    views = [_components(n, edges)]  # no deletion: different connected components never share a block
    for x in range(n):
        views.append(_components(n, [(a, b) for a, b in edges if x not in (a, b)]))
    keys = []
    for a, b in edges:
        if a == b:
            keys.append(None)
            continue
        key = []
        for i, comp in enumerate(views):
            x = i - 1
            key.append(comp[a] if a != x else comp[b])  # a remaining endpoint; both remain connected through e
        keys.append(tuple(key))
    return bridge, first_edge_numbering(keys)


def unit_graphs():
    return json.load(open(os.path.join(GOLDEN, "biconnectivity_unit_graphs.json")))


def test_unit_graphs():
    spec = unit_graphs()
    assert len(spec["bridges"]) >= 8 and len(spec["biconnected_components"]) >= 7
    for case in spec["bridges"]:
        e = np.array(case["edges"], dtype=np.int64).reshape(-1, 2)
        bridge, _ = oracle_biconnectivity(case["n"], e[:, 0], e[:, 1])
        got = sorted(tuple(sorted(p)) for p in e[bridge == 1].tolist())
        if "bridges" in case:
            assert got == sorted(tuple(sorted(p)) for p in case["bridges"]), case["name"]
        assert len(got) == case["bridge_count"], case["name"]
        if case.get("bridge_edge_ids"):
            assert np.nonzero(bridge)[0].tolist() == case["bridge_edge_ids"], case["name"]
    for case in spec["biconnected_components"]:
        e = np.array(case["edges"], dtype=np.int64).reshape(-1, 2)
        _, bcc = oracle_biconnectivity(case["n"], e[:, 0], e[:, 1])
        got = bcc_partition([(c, a, b) for c, (a, b) in zip(bcc.tolist(), e.tolist())])
        exp = bcc_partition([(c, a, b) for c, comp in enumerate(case["components"]) for a, b in comp])
        assert got == exp, case["name"]


def test_e2e_fixtures():
    cases = json.load(open(os.path.join(GOLDEN, "biconnectivity_e2e_cases.json")))["cases"]
    assert sorted(c["module"] for c in cases) == ["biconnected_components", "bridges", "bridges", "bridges"]
    for case in cases:
        dense = {v: i for i, v in enumerate(case["nodes"])}
        e = np.array([(dense[a], dense[b]) for a, b in case["edges"]], dtype=np.int64).reshape(-1, 2)
        bridge, bcc = oracle_biconnectivity(len(dense), e[:, 0], e[:, 1])
        nodes = case["nodes"]
        if case["module"] == "bridges":
            got = sorted((nodes[a], nodes[b]) for a, b in e[bridge == 1].tolist())
            assert got == [(o["from_id"], o["to_id"]) for o in case["output"]], case["name"]
        else:
            got = [(c, nodes[a], nodes[b]) for c, (a, b) in zip(bcc.tolist(), e.tolist())]
            exp = [(o["component"], o["from_id"], o["to_id"]) for o in case["output"]]
            assert bcc_partition(got) == bcc_partition(exp) and len(got) == len(exp), case["name"]


def test_brute_force_definitions():
    rng = np.random.default_rng(17)
    for trial in range(3000):
        n = int(rng.integers(1, 10))
        m = int(rng.integers(0, 16))
        f, t = rng.integers(0, n, m), rng.integers(0, n, m)
        if trial % 3 == 0 and m:  # more multi-edges
            k = int(rng.integers(0, m))
            f, t = np.concatenate([f, t[:k]]), np.concatenate([t, f[:k]])
        bridge, bcc = oracle_biconnectivity(n, f, t)
        exp_bridge, exp_bcc = brute_force(n, f, t)
        assert np.array_equal(bridge, exp_bridge), (n, f.tolist(), t.tolist())
        assert np.array_equal(bcc, exp_bcc), (n, f.tolist(), t.tolist())
    with pytest.raises(AssertionError):
        oracle_biconnectivity(3, [0, 3], [1, 2])  # endpoint out of range
    assert [len(a) for a in oracle_biconnectivity(0, [], [])] == [0, 0]


def test_deep_path_needs_no_call_stack():
    n = 1_000_000
    perm = np.random.default_rng(5).permutation(n)
    bridge, bcc = oracle_biconnectivity(n, perm[:-1], perm[1:])
    assert bridge.all() and np.array_equal(bcc, np.arange(n - 1))
    bridge, bcc = oracle_biconnectivity(n, perm, np.roll(perm, 1))  # one cycle
    assert not bridge.any() and not bcc.any()


def test_matches_the_recorded_reference_module_rows():
    """The reference modules' raw rows on the scattered-gid graphs against the oracle on the same graph view."""
    import test_biconnectivity_modules as bm
    recorded = bm.recorded_rows()["modules"]
    for name in ("bridges", "biconnected_components"):
        graphs = recorded[name]["graphs"]
        assert [c["name"] for c in graphs] == [g[0] for g in bm.scattered_graphs()]
        for (gname, gids, src, dst), call in zip(bm.scattered_graphs(), graphs):
            ref = np.array(call["rows"], dtype=np.int64).reshape(-1, 3)
            ours = bm.module_oracle(name, gids, src, dst)
            if name == "bridges":
                assert len(ref) == len(ours) and bm.same_bridges(ref, ours), gname
            else:
                assert bm.same_components(ref, ours), gname
    assert any(len(c["rows"]) for c in recorded["bridges"]["graphs"])
    sizes = [len(bcc_partition(c["rows"])) for c in recorded["biconnected_components"]["graphs"]]
    assert max(sizes) > 50  # many blocks on the sparse graphs (the dense one is a single block)


@isolated
def test_live_reference_modules():
    """The reference's own modules through the host on random scattered-gid multigraphs, transactional and analytical
    with hidden vertices: the same bridges and the same partition as the oracle."""
    import test_biconnectivity_modules as bm
    if not bm.HAVE_REF_MODULES:
        return  # oracle/_ref/*_reference.so are built only where a reference checkout exists
    rng = np.random.default_rng(41)
    refs = {name: bm.Module(path) for name, path in bm.REF_MODULE_SO.items()}
    bm.check_e2e_fixtures(refs)
    for n, m in [(5, 4), (30, 35), (200, 230), (600, 900)]:
        gids = rng.choice(np.arange(20 * n, dtype=np.int64), size=n, replace=False)
        src, dst = gids[rng.integers(0, n, m)], gids[rng.integers(0, n, m)]
        src, dst = np.concatenate([src, dst[:3]]), np.concatenate([dst, src[:3]])
        hidden = rng.choice(gids, size=max(1, n // 10), replace=False)
        for transactional, hide in ((True, ()), (False, hidden)):
            with bm.Graph(gids, src, dst, transactional=transactional) as g:
                for gid in hide:
                    g.hide_vertex(int(gid))
                rb, rc = refs["bridges"].call(g), refs["biconnected_components"].call(g)
            assert bm.same_bridges(rb, bm.module_oracle("bridges", gids, src, dst, hide)), (n, m)
            assert bm.same_components(rc, bm.module_oracle("biconnected_components", gids, src, dst, hide)), (n, m)
    for module in refs.values():
        module.__exit__()

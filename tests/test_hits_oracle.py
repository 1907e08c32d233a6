"""oracle/cugraph_hits_oracle.c (the checker of the HITS stand-in) against the reference's own e2e fixtures for its cuGraph
HITS module (tests/golden/hits_e2e.json, extracted by tests/golden/make_hits_golden.py from
mage/tests/e2e/hits_test/test_cugraph_*), plus properties of the recurrence.  cuGraph itself is a third-party library
that is absent here; these fixtures (4-6 printed digits) are what pins the restatement.  No GPU."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = json.load(open(os.path.join(REPO, "tests", "golden", "hits_e2e.json")))
HITS_ORACLE_SRC = os.path.join(REPO, "oracle", "cugraph_hits_oracle.c")
HITS_ORACLE_SO = os.path.join(REPO, "oracle", "_build", "libhits_oracle.so")
_oracle = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        if not os.path.exists(HITS_ORACLE_SO) or os.path.getmtime(HITS_ORACLE_SO) < os.path.getmtime(HITS_ORACLE_SRC):
            subprocess.run(["make", "-s", "-C", os.path.join(REPO, "oracle"), "-f", "hits.mk", "oracle"], check=True)
        L = ctypes.CDLL(HITS_ORACLE_SO)
        vp = ctypes.c_void_p
        L.oracle_cugraph_hits.argtypes = [ctypes.c_uint64, ctypes.c_uint64, vp, vp, ctypes.c_uint64, ctypes.c_double,
                                          ctypes.c_int, vp, vp, ctypes.POINTER(ctypes.c_uint64),
                                          ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)]
        _oracle = L
    return _oracle


def oracle_hits(n, f, t, max_iterations=100, tolerance=1e-5, normalized=True):
    """-> (hubs, authorities, iterations, converged)."""
    f = np.ascontiguousarray(f, dtype=np.uint64)
    t = np.ascontiguousarray(t, dtype=np.uint64)
    hubs, auth = np.zeros(max(int(n), 1)), np.zeros(max(int(n), 1))
    it, conv, diff = ctypes.c_uint64(0), ctypes.c_int(0), ctypes.c_double(0.0)
    rc = oracle_lib().oracle_cugraph_hits(int(n), len(f), f.ctypes.data, t.ctypes.data,
                                          int(max_iterations) & (2**64 - 1), float(tolerance), 1 if normalized else 0,
                                          hubs.ctypes.data, auth.ctypes.data, ctypes.byref(it), ctypes.byref(conv),
                                          ctypes.byref(diff))
    if rc:
        raise ValueError(f"oracle_cugraph_hits: {rc}")
    return hubs[:int(n)], auth[:int(n)], it.value, bool(conv.value)


def fixture_arrays(fx):
    """Dense ids in order of first appearance (the module's view sorts by gid; the scores do not depend on the order)."""
    dense = {g: i for i, g in enumerate(fx["nodes"])}
    return dense, [dense[a] for a, _ in fx["edges"]], [dense[b] for _, b in fx["edges"]]


def tolerance_of(fx, want):
    """Printed digits of the value, at least 2e-5 (the solver stops at an L1 residual of N * 1e-5).  The reference's
    printer shows values below 1e-4 as 0.0.  test_cugraph_10_nodes misses its 4 printed digits by up to 2.2e-4 and
    is checked at the reference harness's own ABSOLUTE_TOLERANCE = 1e-3 (mage/tests/e2e/test_module.py)."""
    if fx["name"] == "10_nodes":
        return 1e-3
    if want == 0.0:
        return 1e-4
    digits = len(repr(want).split(".")[1]) if "." in repr(want) else 0
    return max(1.5 * 10.0 ** -digits, 2e-5)


def check_fixture(fx, hubs, auth, dense):
    for gid, want_h, want_a in fx["expected"]:
        got_h, got_a = hubs[dense[gid]], auth[dense[gid]]
        assert abs(got_h - want_h) < tolerance_of(fx, want_h), (fx["name"], gid, "hubs", got_h, want_h)
        assert abs(got_a - want_a) < tolerance_of(fx, want_a), (fx["name"], gid, "authorities", got_a, want_a)


def test_fixture_set_is_complete():
    assert sorted(fx["name"] for fx in FIXTURES) == ["10_nodes", "10_nodes_undirected", "15_nodes", "5_nodes", "empty",
                                                      "networkx_validation"]
    assert all(fx["args"] == [100, 1e-5, True] for fx in FIXTURES)


@pytest.mark.parametrize("fx", FIXTURES, ids=lambda f: f["name"])
def test_reference_e2e_fixtures(fx):
    dense, f, t = fixture_arrays(fx)
    max_iterations, tolerance, normalized = fx["args"]
    hubs, auth, it, conv = oracle_hits(len(dense), f, t, max_iterations, tolerance, normalized)
    assert conv
    if not fx["nodes"]:
        assert fx["expected"] == [] and it == 0
        return
    assert sorted(g for g, _, _ in fx["expected"]) == sorted(dense)  # every fixture vertex has an edge: one row each
    check_fixture(fx, hubs, auth, dense)


def random_multigraph(seed, n=200, m=1500):
    rng = np.random.default_rng(seed)
    f, t = rng.integers(0, n, m), rng.integers(0, n, m)
    f[:20] = t[:20]  # self-loops
    return n, np.concatenate([f, f[:30]]), np.concatenate([t, t[:30]])  # multi-edges


def test_scaling_properties():
    n, f, t = random_multigraph(5)
    hubs, auth, it, conv = oracle_hits(n, f, t, tolerance=1e-10, max_iterations=1000, normalized=False)
    assert conv and hubs.max() == 1.0 and auth.max() == 1.0  # every iterate is scaled by its maximum
    nh, na, it2, conv2 = oracle_hits(n, f, t, tolerance=1e-10, max_iterations=1000, normalized=True)
    assert (it2, conv2) == (it, conv)
    assert abs(nh.sum() - 1.0) < 1e-12 and abs(na.sum() - 1.0) < 1e-12
    assert np.max(np.abs(nh - hubs / hubs.sum())) < 1e-15 and np.max(np.abs(na - auth / auth.sum())) < 1e-15


def test_capped_runs_report_not_converged():
    n, f, t = random_multigraph(6)
    for cap in (1, 2, 7):
        _, _, it, conv = oracle_hits(n, f, t, tolerance=0.0, max_iterations=cap)
        assert it == cap and not conv
    _, _, it, conv = oracle_hits(n, f, t, tolerance=0.0, max_iterations=0)  # 0 runs one iteration
    assert it == 1 and not conv


def test_star_and_complete_bipartite_exact():
    # star 0 -> 1..k: hub 0 alone, every leaf the same authority.  The first iteration reaches the fixed point, the
    # second sees a zero difference.
    k = 7
    hubs, auth, it, conv = oracle_hits(k + 1, [0] * k, list(range(1, k + 1)))
    assert conv and it == 2
    assert hubs.tolist() == [1.0] + [0.0] * k
    assert auth.tolist() == [0.0] + [1.0 / k] * k
    # K_{3,4}: sources 0..2 -> targets 3..6; the same two iterations
    f = [a for a in range(3) for _ in range(4)]
    t = [b for _ in range(3) for b in range(3, 7)]
    hubs, auth, it, conv = oracle_hits(7, f, t, normalized=False)
    assert conv and it == 2
    assert hubs.tolist() == [1.0] * 3 + [0.0] * 4 and auth.tolist() == [0.0] * 3 + [1.0] * 4
    hubs, auth, _, _ = oracle_hits(7, f, t)
    assert hubs.tolist() == [1 / 3] * 3 + [0.0] * 4 and auth.tolist() == [0.0] * 3 + [0.25] * 4


def test_graph_without_edges_gives_zeros():
    hubs, auth, it, conv = oracle_hits(5, [], [])
    assert hubs.tolist() == [0.0] * 5 and auth.tolist() == [0.0] * 5 and it == 0 and conv
    hubs, auth, it, conv = oracle_hits(0, [], [])
    assert len(hubs) == 0 and it == 0 and conv

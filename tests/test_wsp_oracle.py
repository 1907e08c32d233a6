"""oracle/wsp_oracle.c -- the plain-C restatement of the reference's weighted shortest path cursor -- against the
reference's own expectations (tests/golden/wsp_unit_cases.json) and against a brute force over all walks on small
random multigraphs.  No GPU."""
import ctypes
import json
import math
import os
import subprocess

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
WSP_ORACLE_SRC = os.path.join(REPO, "oracle", "wsp_oracle.c")
WSP_ORACLE_SO = os.path.join(REPO, "oracle", "_build", "libwsp_oracle.so")
INT64_MAX = 2**63 - 1
OK, BAD_ARGUMENT, INVALID_WEIGHT, BAD_UPPER_BOUND = 0, 1, 3, 4
_oracle = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        if not os.path.exists(WSP_ORACLE_SO) or os.path.getmtime(WSP_ORACLE_SO) < os.path.getmtime(WSP_ORACLE_SRC):
            subprocess.run(["make", "-s", "-C", os.path.join(REPO, "oracle"), "-f", "wsp.mk", "oracle"], check=True)
        L = ctypes.CDLL(WSP_ORACLE_SO)
        vp = ctypes.c_void_p
        L.oracle_wsp.argtypes = [ctypes.c_uint64, ctypes.c_uint64, vp, vp, vp, ctypes.c_uint64, ctypes.c_int,
                                 ctypes.c_int64, vp, vp, vp, ctypes.POINTER(ctypes.c_uint64)]
        _oracle = L
    return _oracle


def oracle_wsp(n, frm, to, weight, source, direction=0, upper_bound=None):
    """-> (rc, dist float64[n], cursor_depth int32[n], hops int32[n], smallest evaluated invalid COO index or None)."""
    frm = np.ascontiguousarray(frm, dtype=np.uint64)
    to = np.ascontiguousarray(to, dtype=np.uint64)
    w = np.ascontiguousarray(weight, dtype=np.float64)
    dist = np.zeros(max(int(n), 1), dtype=np.float64)
    depth = np.zeros(max(int(n), 1), dtype=np.int32)
    hops = np.zeros(max(int(n), 1), dtype=np.int32)
    invalid = ctypes.c_uint64(0)
    ub = INT64_MAX if upper_bound is None else int(upper_bound)
    rc = oracle_lib().oracle_wsp(int(n), len(frm), frm.ctypes.data, to.ctypes.data, w.ctypes.data, int(source),
                                 int(direction), ub, dist.ctypes.data, depth.ctypes.data, hops.ctypes.data,
                                 ctypes.byref(invalid))
    n = int(n)
    return rc, dist[:n], depth[:n], hops[:n], (None if invalid.value == 2**64 - 1 else invalid.value)


def fixture_cases():
    return json.load(open(os.path.join(GOLDEN, "wsp_unit_cases.json")))["cases"]


def fixture_arrays(case):
    """(from, to, weight) of a fixture; a non-numeric weight becomes NaN (an invalid entry)."""
    e = case["edges"]
    w = [float("nan") if t == "string" else float(x) for _, _, x, t in e]
    return (np.array([a for a, *_ in e], dtype=np.uint64), np.array([b for _, b, *_ in e], dtype=np.uint64),
            np.array(w, dtype=np.float64))


def walked(frm, to, direction):
    """Walked-direction entries (u, x, COO index): out-list first, then in-list, each in COO order."""
    out = []
    if direction != 1:
        out += [(int(a), int(b), e) for e, (a, b) in enumerate(zip(frm, to))]
    if direction != 0:
        out += [(int(b), int(a), e) for e, (a, b) in enumerate(zip(frm, to))]
    return out


def brute_force(n, frm, to, weight, source, direction, upper_bound):
    """The exact left-fold minimum over all walks of at most k edges (k = upper_bound, or n - 1 unbounded: removing a
    cycle never raises a fold, because fl(a + w) is monotone in a and >= a), by enumerating the (vertex, total) pairs of
    walks of exactly j edges.  -> (dist, hops, smallest evaluated invalid index or None)."""
    invalid = [not (w >= 0.0) for w in weight]
    w = [0.0 if (not bad and x == 0.0) else float(x) for x, bad in zip(weight, invalid)]
    entries = walked(frm, to, direction)
    k = max(n - 1, 1) if upper_bound is None else upper_bound
    best = [dict() for _ in range(k + 1)]  # best[j][v] = min over walks of at most j edges
    layer = {(source, 0.0)}
    hop_reach = {source: 0}  # fewest valid edges to reach v
    best[0][source] = 0.0
    for j in range(1, k + 1):
        nxt = set()
        for (u, t) in layer:
            for (a, x, e) in entries:
                if a == u and not invalid[e]:
                    nxt.add((x, t + w[e]))
        layer = nxt
        best[j] = dict(best[j - 1])
        for (x, t) in layer:
            if x not in best[j] or t < best[j][x]:
                best[j][x] = t
            hop_reach.setdefault(x, j)
    expanded = {v for v, h in hop_reach.items() if upper_bound is None or h <= upper_bound - 1}
    bad = [e for (a, _, e) in entries if a in expanded and invalid[e]]
    dist = np.full(n, np.nan)
    hops = np.full(n, -1, dtype=np.int32)
    final = best[k]
    for v, t in final.items():
        if v != source:
            dist[v] = t
    if upper_bound is None:  # BFS depth over tight entries
        d = dict(final)
        level = {source: 0}
        frontier = [source]
        while frontier:
            nf = []
            for u in frontier:
                for (a, x, e) in entries:
                    if a == u and not invalid[e] and x not in level and x in d and d[u] + w[e] == d[x]:
                        level[x] = level[u] + 1
                        nf.append(x)
            frontier = nf
        for v, h in level.items():
            if v != source:
                hops[v] = h
    else:  # smallest j with d_j[v] == d_k[v]
        for v, t in final.items():
            if v != source:
                hops[v] = min(j for j in range(1, k + 1) if best[j].get(v) == t)
    return dist, hops, (min(bad) if bad else None)


def same_bits(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def test_reference_fixtures():
    cases = fixture_cases()
    assert len(cases) == 14
    for case in cases:
        f, t, w = fixture_arrays(case)
        ub = case["upper_bound"]
        rc, dist, depth, hops, invalid = oracle_wsp(case["n"], f, t, w, case["start"], case["direction"], ub)
        if "error" in case:
            kind = case["error"]["kind"]
            assert rc == (BAD_UPPER_BOUND if kind == "upper_bound" else INVALID_WEIGHT), case["name"]
            if kind != "upper_bound":
                bad = [e for e, (_, _, x, ty) in enumerate(case["edges"]) if ty == "string" or x < 0]
                assert invalid == bad[0], case["name"]
            continue
        assert rc == OK, case["name"]
        produced = sorted(v for v in range(case["n"]) if not math.isnan(dist[v]))
        assert produced == sorted(v for v, *_ in case["rows"]), case["name"]
        # the reference yields in order of total: the rows' totals are non-decreasing, and equal ours
        totals = [tot for _, tot, _ in case["rows"]]
        assert totals == sorted(totals), case["name"]
        for v, total, size in case["rows"]:
            assert dist[v] == total, (case["name"], v)
            if size is not None:  # a unique shortest path: every definition agrees with size(le)
                assert depth[v] == size and hops[v] == size, (case["name"], v)
        # the cursor's yield order is by total; our cursor restatement pops in the same order
        order = sorted(produced, key=lambda v: (dist[v], depth[v], v))
        assert [v for v, *_ in case["rows"]] == order, case["name"]


def random_graph(rng):
    n = int(rng.integers(1, 9))
    m = int(rng.integers(0, 15))
    frm, to = rng.integers(0, n, m), rng.integers(0, n, m)
    if m and rng.random() < 0.3:  # a duplicate and a self-loop for certain
        frm = np.concatenate([frm, frm[:1], frm[:1]])
        to = np.concatenate([to, to[:1], frm[:1]])
    pool = [0.0, -0.0, 0.5, 1.0, 2.0, 3.0, 0.1, 0.2, 0.3, 1e-300, 1e16, 2.0**53, math.inf]
    w = np.array([pool[rng.integers(len(pool))] if rng.random() < 0.6 else float(rng.random())
                  for _ in range(len(frm))], dtype=np.float64)
    if len(w) and rng.random() < 0.15:  # invalid entries
        for e in rng.choice(len(w), size=int(rng.integers(1, 3)), replace=True):
            w[e] = math.nan if rng.random() < 0.5 else -float(rng.integers(1, 11))
    if len(w) and rng.random() < 0.15:  # a zero-weight cycle
        frm = np.concatenate([frm, [0, min(1, n - 1)]])
        to = np.concatenate([to, [min(1, n - 1), 0]])
        w = np.concatenate([w, [0.0, 0.0]])
    return n, frm.astype(np.uint64), to.astype(np.uint64), w


def test_equals_brute_force_on_random_multigraphs():
    rng = np.random.default_rng(20261016)
    counts = {"bounded": 0, "unbounded": 0, "invalid": 0, "inf": 0}
    for i in range(2400):
        n, f, t, w = random_graph(rng)
        source = int(rng.integers(0, n))
        direction = i % 3
        ub = [None, 1, 2, 3, 5][(i // 3) % 5]
        rc, dist, depth, hops, invalid = oracle_wsp(n, f, t, w, source, direction, ub)
        bd, bh, binv = brute_force(n, f, t, w, source, direction, ub)
        ctx = (i, n, f.tolist(), t.tolist(), w.tolist(), source, direction, ub)
        assert invalid == binv, ctx
        assert rc == (INVALID_WEIGHT if binv is not None else OK), ctx
        counts["invalid"] += binv is not None
        if binv is not None:
            continue
        assert same_bits(dist, bd), ctx
        assert np.array_equal(hops, bh), ctx
        produced = ~np.isnan(dist)
        assert np.array_equal(depth >= 0, produced) and (depth[produced] >= hops[produced]).all(), ctx
        assert (hops[produced] >= 1).all() and math.isnan(dist[source]), ctx
        counts["bounded" if ub else "unbounded"] += 1
        counts["inf"] += bool(np.isinf(dist).any())
    assert min(counts.values()) >= 20, counts


def test_argument_errors():
    assert oracle_wsp(3, [0], [1], [1.0], 0, 0, 0)[0] == BAD_UPPER_BOUND
    assert oracle_wsp(3, [0], [1], [1.0], 0, 0, -2)[0] == BAD_UPPER_BOUND
    assert oracle_wsp(3, [0], [3], [1.0], 0)[0] == BAD_ARGUMENT
    assert oracle_wsp(3, [0], [1], [1.0], 3)[0] == BAD_ARGUMENT


def test_invalid_edge_evaluation_rules():
    # 0 -> 1 -> 2 -> 3 with an invalid weight on 2 -> 3: evaluated unless the bound stops before vertex 2 is expanded
    f, t = [0, 1, 2, 3], [1, 2, 3, 0]
    w = [1.0, 1.0, -5.0, math.nan]
    assert oracle_wsp(4, f, t, w, 0, 0, 2)[0] == OK  # vertex 2 is at depth 2 == upper_bound: not expanded
    rc, *_, invalid = oracle_wsp(4, f, t, w, 0, 0, 3)
    assert rc == INVALID_WEIGHT and invalid == 2
    # unreachable invalid edge: not an error; reached through IN as well
    rc, dist, *_ = oracle_wsp(5, [0, 3], [1, 4], [2.0, math.nan], 0, 0)
    assert rc == OK and dist[1] == 2.0 and math.isnan(dist[3])
    rc, *_, invalid = oracle_wsp(5, [0, 3, 1], [1, 4, 0], [2.0, math.nan, -1.0], 0, 2)
    assert rc == INVALID_WEIGHT and invalid == 2

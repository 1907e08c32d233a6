"""The algorithms on the BFS device graph (bfs.cu, wsp.cu, wcc.cu, biconnectivity.cu, betweenness.cu) at the list
lengths where their kernels hand work over: 1024-entry warp segments and the out-/in-list join, the top-down /
bottom-up switch at a 1024-vertex frontier, the thread / warp / block walks of WCC's finish and of the bridge sweeps,
betweenness's 512-entry warp / block split, the radix-sort key width around powers of two, and graphs built from
device buffers.  Every graph is built so that the entry sitting on the seam decides the answer: a leaf reached only
through it, a hub joined to its component only by it, the one cross edge that makes a tree edge a non-bridge, a vertex
whose sigma comes only through a 512-entry list.  Integers and totals must equal the oracles exactly, betweenness within
test_bc_module.assert_matches.  Each case also asserts the degree or the run statistic that shows it reached its seam."""
import ctypes

import numpy as np
import pytest

import memgraph_b200 as mg
from _checkers import BfsOracle
from test_bc_module import assert_matches
from test_bc_oracle import oracle_bc
from test_biconnectivity_oracle import oracle_biconnectivity
from test_wcc_oracle import oracle_wcc
from test_wsp_oracle import oracle_wsp, same_bits

pytestmark = pytest.mark.gpu

OUT, IN, BOTH = 0, 1, 2
INT64_MAX = 2**63 - 1
SEG_DEGREES = (1, 1023, 1024, 1025, 2047, 2048, 2049, 3073)
JOINS = (1023, 1024, 1025)  # out-list lengths of a BOTH list


@pytest.fixture(scope="module")
def lib():
    from memgraph_b200 import _native as N
    return N


class Coo:
    """COO edges with weights, added as arcs of the direction a run walks: an OUT arc u -> v is the edge (u, v), an IN
    arc is the edge (v, u); BOTH takes the side explicitly ("out": (u, v) sits in u's out-list, "in": (v, u) in its
    in-list)."""

    def __init__(self, direction):
        self.direction, self.f, self.t, self.w = direction, [], [], []

    def arc(self, u, v, w=1.0, side="out", copies=1):
        reverse = self.direction == IN or (self.direction == BOTH and side == "in")
        a, b = (v, u) if reverse else (u, v)
        self.f += [a] * copies
        self.t += [b] * copies
        self.w += [w] * copies

    def arrays(self):
        return np.array(self.f, dtype=np.uint64), np.array(self.t, dtype=np.uint64), np.array(self.w, dtype=np.float64)


def walked_degree(n, f, t, direction):
    out = np.bincount(f.astype(np.int64), minlength=n)
    inn = np.bincount(t.astype(np.int64), minlength=n)
    return {OUT: out, IN: inn, BOTH: out + inn}[direction]


def segment_ladder(direction, backup):
    """Source 0 -> one hub per list length -> a distinct leaf per entry of the hub's walked list, leaf ids rising
    with the entry's position, so each entry (position 0, k * 1024 - 1, k * 1024, the out/in join, the last one) is
    the only way to its leaf.  In BOTH the source is the hub's out-list entry 0 (edge hub -> source) and the hub's out
    list is 1023, 1024 or 1025 long, the rest of it in the in-list.  Hub entry k weighs 1 + k % 16.  `backup` adds
    vertex 1 (total 0.5) with an arc of weight 64 to every leaf: dropping a hub entry then gives a heavier total
    instead of an unreached leaf.  -> (n, f, t, w, {hub: walked length})."""
    g = Coo(direction)
    nxt = 2 if backup else 1
    specs = [(d, d) for d in SEG_DEGREES] if direction != BOTH else \
        sorted({(d, min(a, d)) for d in SEG_DEGREES for a in JOINS})
    hubs, leaves = {}, []
    for degree, out_len in specs:
        hub = nxt
        nxt += 1
        hubs[hub] = degree
        if direction == BOTH:
            g.arc(0, hub, 1.0, side="in")  # the edge (hub, 0): the source is entry 0 of the hub's out-list
            sides = ["out"] * (out_len - 1) + ["in"] * (degree - out_len)
        else:
            g.arc(0, hub, 1.0)
            sides = ["out"] * degree
        for k, side in enumerate(sides, start=1 if direction == BOTH else 0):
            g.arc(hub, nxt, 1.0 + k % 16, side=side)
            leaves.append(nxt)
            nxt += 1
    if backup:
        g.arc(0, 1, 0.5)
        for leaf in leaves:
            g.arc(1, leaf, 64.0)
    f, t, w = g.arrays()
    return nxt, f, t, w, hubs


@pytest.mark.parametrize("direction", [OUT, IN, BOTH])
def test_bfs_segments(direction):
    from memgraph_b200 import bfs
    oracle = BfsOracle()
    n, f, t, _, hubs = segment_ladder(direction, backup=False)
    deg = walked_degree(n, f, t, direction)
    assert all(deg[h] == d for h, d in hubs.items())
    with bfs.BfsGraph(n, f, t) as g:
        for lower, upper in [(1, INT64_MAX), (2, 2), (1, 1), (2, 3), (3, INT64_MAX)]:
            got, st = g.distances(0, direction, lower, upper)
            ref = oracle.distances(n, f, t, 0, direction, lower, upper)
            assert np.array_equal(got.astype(np.int64), ref), (direction, lower, upper)
            if upper == INT64_MAX and lower == 1:
                assert (got[1:] > 0).all() and st["reached"] == n - 1
                # levels 0 and 1 (frontiers of 1 and of the hubs) go top-down, so the hubs' lists are cut in segments;
                # in BOTH the leaves' level may go bottom-up
                assert st["top_down_levels"] >= 2 and st["bottom_up_levels"] <= (direction == BOTH)


@pytest.mark.parametrize("direction", [OUT, IN, BOTH])
def test_wsp_segments(direction):
    from memgraph_b200 import bfs
    n, f, t, w, hubs = segment_ladder(direction, backup=True)
    deg = walked_degree(n, f, t, direction)
    assert all(deg[h] == d for h, d in hubs.items())
    with bfs.BfsGraph(n, f, t) as g:
        g.set_weights(f, t, w)
        for ub in (None, 1, 2):
            rc, dist, _, hops, _ = oracle_wsp(n, f, t, w, 0, direction, ub)
            assert rc == 0
            gd, gh, st = g.weighted_distances(0, direction, ub)
            assert same_bits(gd, dist) and np.array_equal(gh, hops), (direction, ub)
            if ub != 1:
                leaves = np.setdiff1d(np.arange(2, n), list(hubs))
                assert (dist[leaves] < 64).all()  # every leaf's total comes through its hub entry
                assert st["reached"] == n - 1


@pytest.mark.parametrize("direction", [OUT, IN, BOTH])
@pytest.mark.parametrize("children", [1024, 1025])
def test_bfs_switches_to_bottom_up_above_1024_frontier_vertices(direction, children):
    """Source 0 -> children 1..K, child i -> grandchild K + i twice, so the children's edges far outnumber 1/14 of the
    unexplored ones; only the frontier size keeps K = 1024 top-down."""
    from memgraph_b200 import bfs
    oracle = BfsOracle()
    g = Coo(direction)
    for i in range(1, children + 1):
        g.arc(0, i)
        g.arc(i, children + i, copies=2)
    f, t, _ = g.arrays()
    n = 2 * children + 1
    with bfs.BfsGraph(n, f, t) as h:
        for lower, upper in [(1, INT64_MAX), (2, 2), (1, 1)]:
            got, st = h.distances(0, direction, lower, upper)
            assert np.array_equal(got.astype(np.int64), oracle.distances(n, f, t, 0, direction, lower, upper))
            if upper == INT64_MAX:
                assert (got[1:children + 1] == 1).all() and (got[children + 1:] == 2).all()
                if children == 1024:
                    assert st["bottom_up_levels"] == 0 and st["top_down_levels"] == 3
                else:
                    assert st["bottom_up_levels"] >= 1


WCC_DEGREES = (2, 3, 18, 19, 4098, 4099)  # remaining entries after 2 sample rounds: 0, 1, 16, 17, 4096, 4097


def wcc_ladder(path=20000):
    """A doubled path v -> v + 1 (twice) over the top `path` ids is the giant component; its vertices' sampled entries are
    their path neighbours, so a hub's edge lands at position >= 2 of theirs.  Below it, small components of hub h:
      first  h -> a twice, h -> x, b -> h (D - 3 times): h's list is [a, a, x, b, ...]; its one link to the giant (x)
             is position 2, the first entry the finish walks;
      last   h -> a (D - 1 times), h -> y: its one link to the giant (y) is its last entry.
    -> (n, f, t, {hub: degree}, giant's first id)."""
    f, t = [], []
    hubs = {}
    nxt = 0
    cases = [(d, "first") for d in WCC_DEGREES if d >= 3] + [(d, "last") for d in WCC_DEGREES]
    plan = []
    for d, kind in cases:
        h, a, b = nxt, nxt + 1, nxt + 2
        nxt += 3
        hubs[h] = d
        plan.append((d, kind, h, a, b))
    q = nxt
    for i, (d, kind, h, a, b) in enumerate(plan):
        giant_member = q + 1000 + 37 * i
        if kind == "first":
            f += [h, h, h] + [b] * (d - 3)
            t += [a, a, giant_member] + [h] * (d - 3)
        else:
            f += [h] * d
            t += [a] * (d - 1) + [giant_member]
    v = np.arange(q, q + path - 1)
    f = np.concatenate([np.array(f, dtype=np.int64), v, v])
    t = np.concatenate([np.array(t, dtype=np.int64), v + 1, v + 1])
    return q + path, f.astype(np.uint64), t.astype(np.uint64), hubs, q


def sampled_giant(n, f, t, first_giant):
    """The vertices that wcc.cu's two sample rounds join to the giant's vertex `first_giant`: every vertex linked with
    entries 0 and 1 of its undirected list (sorted out-list, then sorted in-list)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    f64, t64 = f.astype(np.int64), t.astype(np.int64)
    out = np.lexsort((t64, f64))
    inn = np.lexsort((f64, t64))
    od, idg = np.bincount(f64, minlength=n), np.bincount(t64, minlength=n)
    optr, iptr = np.concatenate([[0], np.cumsum(od)]), np.concatenate([[0], np.cumsum(idg)])
    a, b = [], []
    for r in (0, 1):
        for v in np.nonzero(od + idg > r)[0]:
            w = t64[out[optr[v] + r]] if r < od[v] else f64[inn[iptr[v] + r - od[v]]]
            a.append(v)
            b.append(w)
    _, label = connected_components(coo_matrix((np.ones(len(a)), (a, b)), shape=(n, n)), directed=False)
    return label == label[first_giant]


def test_wcc_finish_walks_thread_warp_and_block_lists():
    from memgraph_b200 import connectivity as cc
    n, f, t, hubs, first_giant = wcc_ladder()
    deg = walked_degree(n, f, t, BOTH)
    assert all(deg[h] == d for h, d in hubs.items())
    giant = sampled_giant(n, f, t, first_giant)
    assert not giant[[h for h, d in hubs.items() if d >= 3]].any()  # these hubs are left to the finish
    exp = oracle_wcc(n, f, t)
    with cc.BfsGraph(n, f, t) as g:
        got, stats = cc.wcc_run(g)
    assert np.array_equal(got, exp)
    assert stats["skipped_vertices"] == int(giant.sum())
    # every hub ends in the giant component, through exactly one entry
    assert (exp[list(hubs)] == exp[first_giant]).all()
    assert np.array_equal(cc.weakly_connected_components(n, f, t), exp)


BRIDGE_DEGREES = (16, 17, 4096, 4097)  # thread, warp, warp, block


def bridge_ladder():
    """One component per (degree, case), hub h with exactly `degree` undirected entries and degree - 2 (or - 3) pendant
    leaves; r is each component's smallest id, so the forest's root:
      first         r - P, r - Q, P -> h (in-list), h -> Q (out-list entry 0): Q is the one cross edge that makes
                    (P, h) and the cycle r P h Q a non-bridge, and it is h's first entry
      last          the same with h -> P (out-list) and Q -> h, Q the largest id: Q is h's last entry
      parallel_lo   r - P, h -> P and P -> h: the doubled tree edge is at h's out-list position 0 and in-list position 0
      parallel_hi   the same with P the largest id: the end of h's out-list and the end of its in-list
    -> (n, f, t, {hub: degree})."""
    f, t = [], []
    hubs = {}
    base = 0
    for d in BRIDGE_DEGREES:
        for case in ("first", "last", "parallel_lo", "parallel_hi"):
            r = base
            if case == "first":
                p, q, h = base + 1, base + 2, base + 3
                leaves = list(range(base + 4, base + 4 + d - 2))
                f += [r, r, p, h] + [h] * len(leaves)
                t += [p, q, h, q] + leaves
                end = leaves[-1] + 1
            elif case == "last":
                p, h = base + 1, base + 2
                leaves = list(range(base + 3, base + 3 + d - 2))
                q = leaves[-1] + 1
                half = len(leaves) // 2
                f += [r, r, h, q] + [h] * half + leaves[half:]
                t += [p, q, p, h] + leaves[:half] + [h] * (len(leaves) - half)
                end = q + 1
            elif case == "parallel_lo":
                p, h = base + 1, base + 2
                leaves = list(range(base + 3, base + 3 + d - 2))
                half = len(leaves) // 2
                f += [r, h, p] + [h] * half + leaves[half:]
                t += [p, p, h] + leaves[:half] + [h] * (len(leaves) - half)
                end = leaves[-1] + 1
            else:
                h = base + 1
                leaves = list(range(base + 2, base + 2 + d - 2))
                p = leaves[-1] + 1
                half = len(leaves) // 2
                f += [r, h, p] + [h] * half + leaves[half:]
                t += [p, p, h] + leaves[:half] + [h] * (len(leaves) - half)
                end = p + 1
            hubs[h] = d
            base = end
    return base, np.array(f, dtype=np.uint64), np.array(t, dtype=np.uint64), hubs


def test_bridges_and_blocks_at_the_walk_splits():
    from memgraph_b200 import connectivity as cc
    n, f, t, hubs = bridge_ladder()
    deg = walked_degree(n, f, t, BOTH)
    assert all(deg[h] == d for h, d in hubs.items())
    exp_bridge, exp_bcc = oracle_biconnectivity(n, f, t)
    with cc.BfsGraph(n, f, t) as g:
        bridge, bcc, stats = cc.biconnectivity_run(g, f, t)
    assert np.array_equal(bridge, exp_bridge)
    assert np.array_equal(bcc, exp_bcc)
    # the decisive entries: no edge at a hub is a bridge except its pendant leaves' (and r - P in the parallel cases)
    leaves_per_hub = [d - 2 for d in hubs.values()]
    parallel_roots = 2 * len(BRIDGE_DEGREES)
    assert stats["bridges"] == int(exp_bridge.sum()) == sum(leaves_per_hub) + parallel_roots
    assert stats["trees"] == 4 * len(BRIDGE_DEGREES)


def bc_ladder(directed):
    """Per list length D in (512, 513): an in-hub h whose pulled list is exactly D long (a -> u_i -> h -> z) and an
    out-hub g whose pushed list is exactly D long (c -> g -> x_i -> y).  Undirected, both lists are the undirected one,
    so one of the D entries is the path's other end.  -> (n, f, t, {hub: pulled or pushed length})."""
    f, t = [], []
    hubs = {}
    nxt = 0
    for d in (512, 513):
        k = d if directed else d - 1
        a, h, z = nxt, nxt + 1, nxt + 2
        u = list(range(nxt + 3, nxt + 3 + k))
        nxt = u[-1] + 1
        f += [a] * k + u + [h]
        t += u + [h] * k + [z]
        hubs[("in", h)] = d
        c, g, y = nxt, nxt + 1, nxt + 2
        x = list(range(nxt + 3, nxt + 3 + k))
        nxt = x[-1] + 1
        f += [c] + [g] * k + x
        t += [g] + x + [y] * k
        hubs[("out", g)] = d
    return nxt, np.array(f, dtype=np.uint64), np.array(t, dtype=np.uint64), hubs


@pytest.mark.parametrize("directed", [True, False])
def test_betweenness_at_512_pulled_and_pushed_entries(directed):
    from memgraph_b200 import betweenness as bc
    n, f, t, hubs = bc_ladder(directed)
    out_deg = walked_degree(n, f, t, OUT if directed else BOTH)
    in_deg = walked_degree(n, f, t, IN if directed else BOTH)
    for (side, v), d in hubs.items():
        assert (in_deg if side == "in" else out_deg)[v] == d
    ref = oracle_bc(n, f, t, directed, False)
    with bc.BfsGraph(n, f, t) as g:
        got, stats = bc.bc_range(g, directed)
    assert stats["sources"] == n
    assert_matches(got, ref)
    assert all(ref[v] > 0 for (_, v) in hubs)  # every hub lies on paths, so its list decides its value
    assert_matches(bc.betweenness_centrality(n, f, t, directed, True), oracle_bc(n, f, t, directed, True))


@pytest.mark.parametrize("n", [2**16 - 1, 2**16, 2**16 + 1, 2**17 + 1])
def test_sort_key_width_around_powers_of_two(n):
    """(row << 32 | col) keys are sorted on 32 + bits(n) bits: edges at vertex n - 1 (as row and as column) and at 0."""
    from memgraph_b200 import betweenness as bcm
    from memgraph_b200 import bfs
    from memgraph_b200 import connectivity as cc
    rng = np.random.default_rng(n)
    m = 2 * n
    f = np.concatenate([rng.integers(0, n, m), [0, n - 1, n - 1, n - 2, n - 1, 0]]).astype(np.uint64)
    t = np.concatenate([rng.integers(0, n, m), [n - 1, 0, n - 2, n - 1, n - 1, n - 1]]).astype(np.uint64)
    w = bfs.splitmix_weights(len(f))
    oracle = BfsOracle()
    with bfs.BfsGraph(n, f, t) as g:
        for source in (0, n - 1):
            for direction in (OUT, IN, BOTH):
                got, _ = g.distances(source, direction)
                assert np.array_equal(got.astype(np.int64), oracle.distances(n, f, t, source, direction))
        g.set_weights(f, t, w)
        for source, direction, ub in [(n - 1, OUT, None), (0, BOTH, None), (n - 1, IN, 2)]:
            rc, dist, _, hops, _ = oracle_wsp(n, f, t, w, source, direction, ub)
            gd, gh, _ = g.weighted_distances(source, direction, ub)
            assert rc == 0 and same_bits(gd, dist) and np.array_equal(gh, hops), (source, direction, ub)
        comp, _ = cc.wcc_run(g)
        assert np.array_equal(comp, oracle_wcc(n, f, t))
        bridge, bcc, _ = cc.biconnectivity_run(g, f, t)
        exp_bridge, exp_bcc = oracle_biconnectivity(n, f, t)
        assert np.array_equal(bridge, exp_bridge) and np.array_equal(bcc, exp_bcc)
        for directed, (lo, hi) in [(True, (n - 32, n)), (False, (0, 32))]:
            got, _ = bcm.bc_range(g, directed, lo, hi)
            assert_matches(got, oracle_bc(n, f, t, directed, False, lo, hi))


def test_device_built_graph_equals_host_built(lib):
    """BfsGraph.from_device on mg.rmat_edges_device buffers against the host-built handle, byte for byte; an endpoint
    one past the vertex count is refused on the device; device-resident outputs equal the host-output calls."""
    import torch
    from memgraph_b200 import betweenness as bcm
    from memgraph_b200 import bfs
    from memgraph_b200 import connectivity as cc
    scale = 14
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    w = bfs.splitmix_weights(m)
    L = lib.lib()
    d_f, d_t = lib.vp(), lib.vp()
    assert L.mgb200_device_malloc(0, 4 * m, ctypes.byref(d_f)) == 0
    assert L.mgb200_device_malloc(0, 4 * m, ctypes.byref(d_t)) == 0
    try:
        mg.rmat_edges_device(scale, m, d_f, d_t)
        # a vertex count equal to the largest endpoint leaves exactly that endpoint out of range (the generator does
        # not permute ids, so vertex 2^scale - 1 itself almost never occurs)
        top = int(max(f.max(), t.max()))
        h = lib.vp()
        rc = L.mgb200_bfs_graph_create_device(0, top, m, d_f, d_t, ctypes.byref(h))
        assert rc == lib.ERR_INVALID_ARGUMENT and not h.value
        assert b"edge endpoint out of range" in L.mgb200_last_error()
        with pytest.raises(mg.MgB200Error, match="edge endpoint out of range"):
            bfs.BfsGraph.from_device(top, m, d_f, d_t)
        dev = bfs.BfsGraph.from_device(n, m, d_f, d_t)
    finally:
        L.mgb200_device_free(0, d_f)
        L.mgb200_device_free(0, d_t)
    with dev, bfs.BfsGraph(n, f, t) as host:
        for source in (0, 1, n - 1):
            for direction in (OUT, IN, BOTH):
                a, _ = dev.distances(source, direction)
                b, _ = host.distances(source, direction)
                assert a.tobytes() == b.tobytes(), (source, direction)
        dev.set_weights(f, t, w)
        host.set_weights(f, t, w)
        for direction, ub in [(OUT, None), (IN, None), (BOTH, None), (BOTH, 2)]:
            a = dev.weighted_distances(0, direction, ub)
            b = host.weighted_distances(0, direction, ub)
            assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), (direction, ub)
        assert cc.wcc_run(dev)[0].tobytes() == cc.wcc_run(host)[0].tobytes()
        a, b = cc.biconnectivity_run(dev, f, t), cc.biconnectivity_run(host, f, t)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
        for directed, lo, hi in [(True, 0, 64), (False, 100, 164)]:
            a, _ = bcm.bc_range(dev, directed, lo, hi)
            b, _ = bcm.bc_range(host, directed, lo, hi)
            assert a.tobytes() == b.tobytes(), directed
        # device-resident outputs
        st = lib.BfsStats()
        for direction in (OUT, BOTH):
            out = torch.full((n,), -7, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()  # the library writes on its own stream
            assert L.mgb200_bfs_run(dev._h, 0, direction, 1, INT64_MAX, out.data_ptr(), 1, ctypes.byref(st)) == 0
            assert out.cpu().numpy().tobytes() == dev.distances(0, direction)[0].tobytes()
        bc_dev = torch.full((n,), -1.0, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        assert L.mgb200_bc_run(dev._h, 1, 0, 64, lib.ABORT_FN(), None, bc_dev.data_ptr(), 1,
                               ctypes.byref(lib.BcStats())) == 0
        assert bc_dev.cpu().numpy().tobytes() == bcm.bc_range(dev, True, 0, 64)[0].tobytes()

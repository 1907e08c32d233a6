"""Maximum bipartite matching (memgraph_b200/csrc/bipartite_matching.cu) where its kernels hand work over or stop: a
phase search walking a hub's list from a level-2 frontier at the thread / warp / block walk lengths (16 / 4096
entries), the greedy rounds' cap of 4 and their stop after a round that adds nothing, augmenting paths thousands of
levels deep, trees that compete for one vertex, and one BfsGraph shared by every algorithm built on it.  Every graph is
built so that one entry, one round or one tree decides the answer, and each case asserts the run statistic that shows
the run reached it.  The builders are checked without a GPU against the lists as the device graph orders them, a numpy
model of the greedy rule and the C oracle, so each decision is known to sit on its seam before a kernel runs it."""
import functools

import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components, shortest_path

from test_bipartite_oracle import bipartite_rmat, oracle_matching
from test_gpu_bipartite import certify, check

OUT, IN, BOTH = 0, 1, 2
GREEDY_ROUNDS = 4  # kGreedyRounds
WALK_DEGREES = (16, 17, 4096, 4097, 40000)  # a thread walks up to 16 entries, a warp up to 4096, a block above
POSITIONS = (1, 15, 16, 31, 32, 255, 256)
STAIRS = (1, 3, 4, 5, 6, 100)
PATHS = (1, 2, 1000, 5000)
SCATTERED = (1, 2, 3, 7, 64, 301, 1000, 2500)


@pytest.fixture(scope="module")
def mm():
    from memgraph_b200 import matching
    return matching


def no_ms(stats):
    return {k: v for k, v in stats.items() if not k.endswith("_ms")}


# ---- host model ------------------------------------------------------------------------------------------------------

def undirected_lists(n, f, t):
    """Every vertex's list as the device walks it: its out-list sorted by target, then its in-list sorted by source.
    -> (ptr int64[n + 1], adj int64[2m])."""
    f, t = np.asarray(f, dtype=np.int64), np.asarray(t, dtype=np.int64)
    owner, other = np.concatenate([f, t]), np.concatenate([t, f])
    side = np.repeat([0, 1], len(f))
    ptr = np.concatenate([[0], np.cumsum(np.bincount(owner, minlength=n))])
    return ptr, other[np.lexsort((other, side, owner))]


def colouring(n, f, t):
    """Forest depth of every vertex, from its component's smallest id (a bipartite graph's breadth-first levels)."""
    f, t = np.asarray(f, dtype=np.int64), np.asarray(t, dtype=np.int64)
    _, label = connected_components(coo_matrix((np.ones(len(f)), (f, t)), shape=(n, n)), directed=False)
    root = np.full(label.max() + 1, n)
    np.minimum.at(root, label, np.arange(n))
    a, b = np.concatenate([f, np.full(len(root), n)]), np.concatenate([t, root])  # vertex n joined to every root
    hops = shortest_path(coo_matrix((np.ones(len(a)), (a, b)), shape=(n + 1, n + 1)).tocsr(), directed=False,
                         unweighted=True, indices=n)
    return hops[:n].astype(np.int64) - 1


def greedy(n, f, t):
    """The greedy rounds as bipartite_matching.cu states them: L = the even forest depths; every free L vertex proposes
    to its smallest free neighbour and every R vertex accepts its smallest proposer; at most GREEDY_ROUNDS rounds, and
    none after a round that adds nothing.  -> (mate int64[n], pairs made by each round that ran)."""
    ptr, adj = undirected_lists(n, f, t)
    owner = np.repeat(np.arange(n), np.diff(ptr))
    left = colouring(n, f, t) % 2 == 0
    mate = np.full(n, -1, dtype=np.int64)
    added = []
    while len(added) < GREEDY_ROUNDS:
        free = left & (mate < 0)
        if not free.any():
            break
        live = free[owner] & (mate[adj] < 0)
        target = np.full(n, n)
        np.minimum.at(target, owner[live], adj[live])
        u = np.flatnonzero(target < n)
        proposer = np.full(n, n)
        np.minimum.at(proposer, target[u], u)
        won = u[proposer[target[u]] == u]
        mate[won], mate[target[won]] = target[won], won
        added.append(len(won))
        if not len(won):
            break
    return mate, added


def assert_matching(n, f, t, mate, size):
    """mate pairs `size` edges of the graph, each vertex at most once."""
    v = np.flatnonzero(mate >= 0)
    assert len(v) == 2 * size and (mate[mate[v]] == v).all()
    edges = set(zip(np.asarray(f).tolist(), np.asarray(t).tolist()))
    assert all((a, b) in edges or (b, a) in edges for a, b in zip(v.tolist(), mate[v].tolist()))


# ---- builders --------------------------------------------------------------------------------------------------------

def hub_gadget(degree, position, copies=1, out_len=None, base=0):
    """Hub H = base, the component's smallest id (so the root, on the L side), with an undirected list of `degree`
    entries: entry 0 is r0, entries [position, position + copies) are copies of r*, every other entry is its own r_i.
    a0's only neighbour is r0, each r_i has a leaf l_i of its own, and r* has no neighbour but H.  Entries
    [0, out_len) are H's out-list (edges H -> x), the rest its in-list (x -> H); ids rise with the entry, so both halves
    are sorted as the device keeps them.  Greedy round 0 pairs H - r0 (H < a0) and every l_i - r_i, and round 1 finds
    nothing for a0.  Phase 1 then walks a0 -> r0 -> H and reaches H's whole list from a level-2 frontier; its search
    ends, and the answer gains its last pair, only through an entry of r*.
    -> dict(n = one past the largest id, f, t, hub, a0, r0, rstar, pairs = the maximum, and the arguments)."""
    out_len = degree if out_len is None else out_len
    entry = np.arange(degree)
    nbr = base + 1 + entry - np.clip(entry - position, 0, copies - 1)  # ids in entry order, one for r*'s copies
    rstar = base + 1 + position
    others = nbr[1:][nbr[1:] != rstar]
    a0 = int(nbr[-1]) + 1
    leaves = a0 + 1 + np.arange(len(others))
    out = entry < out_len
    f = np.concatenate([np.where(out, base, nbr), [a0], others])
    t = np.concatenate([np.where(out, nbr, base), [nbr[0]], leaves])
    return dict(n=int(a0 + 1 + len(others)), f=f.astype(np.uint64), t=t.astype(np.uint64), hub=base, a0=a0,
                r0=int(nbr[0]), rstar=int(rstar), pairs=len(others) + 2, degree=degree, position=position,
                copies=copies, out_len=out_len)


def gadget_specs(degree):
    """(name, position of r*, copies, out-list length) of every gadget with a hub list of `degree` entries."""
    half = degree // 2
    positions = sorted({p for p in POSITIONS + (degree - 1,) if p < degree})
    return ([(f"out@{p}", p, 1, degree) for p in positions] + [(f"in@{p}", p, 1, 0) for p in positions] +
            [("last_out", half - 1, 1, half), ("first_in", half, 1, half),
             ("multi_across_join", half - 1, 3, half), ("multi_at_end", degree - 3, 3, degree)])


def gadgets(degrees):
    """Every gadget of `degrees`, with disjoint ids.  -> (name, gadget dict) list."""
    out, base = [], 0
    for d in degrees:
        for name, p, c, o in gadget_specs(d):
            g = hub_gadget(d, p, c, o, base)
            out.append((f"D{d}:{name}", g))
            base = g["n"]
    return out


@functools.lru_cache(maxsize=None)
def all_gadgets():
    """Every gadget of every walk length in one graph.  -> (n, f, t, gadget list)."""
    parts = gadgets(WALK_DEGREES)
    f = np.concatenate([g["f"] for _, g in parts])
    t = np.concatenate([g["t"] for _, g in parts])
    return parts[-1][1]["n"], f, t, parts


def staircase(k):
    """L_i = i adjacent to R_0 .. R_i (R_j = k + j): round r pairs L_r - R_r and nothing else, so the greedy rounds
    make min(k, 4) pairs and phase 1 the rest at once (R_j's smallest frontier neighbour is L_j).  -> (n, f, t)."""
    i, j = np.tril_indices(k)
    return 2 * k, i.astype(np.uint64), (k + j).astype(np.uint64)


STAR_SIZES = (2, 5, 40)


def stars():
    """Per size s: an R hub with s leaves, the first leaf its component's smallest id.  Round 0 pairs every hub with its
    first leaf, and that is already maximum; round 1 finds no free neighbour for the other leaves.  They stay free and
    the cap is two rounds away, so only the stop after a fruitless round ends the rounds.  -> (n, f, t)."""
    f, t, base = [], [], 0
    for s in STAR_SIZES:
        hub = base + 1
        leaves = [base] + list(range(base + 2, base + s + 1))
        f += [hub] * s
        t += leaves
        base += s + 1
    return base, np.array(f, dtype=np.uint64), np.array(t, dtype=np.uint64)


def path_ids(k):
    """Ids of v0 .. v_{2k+1} along a path: even positions k, k - 1, .., 0 and odd positions k + 1, .., 2k + 1.  Each
    v_{2i} proposes to v_{2i-1} (smaller than v_{2i+1}) and wins it against v_{2i-2}, so the greedy rounds match every
    middle edge and leave one augmenting path v0 .. v_{2k+1}, found at search level k + 1."""
    ids = np.empty(2 * k + 2, dtype=np.int64)
    ids[0::2] = np.arange(k, -1, -1)
    ids[1::2] = np.arange(k + 1, 2 * k + 2)
    return ids


def path_edges(ids):
    return ids[:-1].astype(np.uint64), ids[1:].astype(np.uint64)


def scattered_paths(lengths, seed):
    """Disjoint augmenting paths (path_ids' order) whose ids are drawn at random from one range: in each path the even
    positions' ids still fall along it and the odd positions' rise (all the greedy rounds need), and its smallest id
    is v_{2k}, but the two sides and the paths interleave, and each edge's orientation is random.
    -> (n, f, t, list of each path's ids in path order)."""
    rng = np.random.default_rng(seed)
    n = sum(2 * k + 2 for k in lengths)
    perm = rng.permutation(n)
    paths, at = [], 0
    for k in lengths:
        chunk = np.sort(perm[at:at + 2 * k + 2])
        at += 2 * k + 2
        even = np.zeros(2 * k + 1, dtype=bool)
        even[rng.choice(2 * k + 1, size=k, replace=False)] = True
        ids = np.empty(2 * k + 2, dtype=np.int64)
        ids[0::2] = np.concatenate([chunk[:1], chunk[1:][even]])[::-1]
        ids[1::2] = chunk[1:][~even]
        paths.append(ids)
    f = np.concatenate([p[:-1] for p in paths])
    t = np.concatenate([p[1:] for p in paths])
    flip = rng.random(len(f)) < 0.5
    return n, np.where(flip, t, f).astype(np.uint64), np.where(flip, f, t).astype(np.uint64), paths


def path_mate(n, paths):
    """The matching after the augmentation: v_{2i} - v_{2i+1} on every path."""
    mate = np.full(n, -1, dtype=np.int64)
    for ids in paths:
        mate[ids[0::2]], mate[ids[1::2]] = ids[1::2], ids[0::2]
    return mate


# Two free roots A = 3 and B = 4 reach the matched r = 1 at level 1.  pred[r] = min(A, B), so A's tree takes r and its
# mate m = 0, whose free s = 2 ends the path A - r - m - s; B's phase-2 search dies at r.  Greedy: m wins r from A and
# B (m proposes r < s).
TWO_ROOTS = dict(n=5, f=[0, 0, 3, 4], t=[1, 2, 1, 1], greedy=[1, 0, -1, -1, -1], mate=[2, 3, 0, 1, -1],
                 initial=1, matched=2, phases=2, max_levels=2)
# m = 0, c = 1, a = 2, b = 3 on L; r = 4, x = 5, s1 = 6, s2 = 7 on R.  Greedy: m - r, c - x.  Phase 1 from a and b:
# level 2 is m (tree a) and c (tree b); s1 is both m's and c's, and pred[s1] = min(m, c) = m, so both free s1 and s2
# fall to tree a, whose end is the smaller, s1: a - r, m - s1.  Phase 2 from b: b - x - c - s1 - m - {r, s2} at level
# 3; s2 ends it, and a (r's mate) does not join, the tree having an end.  Phase 3 has no free root.
TWO_ENDS = dict(n=8, f=[0, 0, 0, 2, 1, 1, 3], t=[4, 6, 7, 4, 5, 6, 5], greedy=[4, 5, -1, -1, 0, 1, -1, -1],
                mate=[7, 6, 4, 5, 2, 3, 1, 0], initial=2, matched=4, phases=3, max_levels=3)


# ---- builders on the host --------------------------------------------------------------------------------------------

def test_gadgets_put_r_star_on_the_seam():
    n, f, t, parts = all_gadgets()
    assert len({name for name, _ in parts}) == len(parts)
    for name, g in parts:
        h = g["hub"]
        ptr, adj = undirected_lists(g["n"], g["f"], g["t"])
        lst = adj[ptr[h]:ptr[h + 1]]
        assert len(lst) == g["degree"] and lst[0] == g["r0"] == lst.min() and h < g["a0"], name
        assert np.array_equal(np.flatnonzero(lst == g["rstar"]), g["position"] + np.arange(g["copies"])), name
        assert int((g["f"] == h).sum()) == g["out_len"], name  # r*'s side: out-list entries [0, out_len)
        mate, added = greedy(g["n"], g["f"], g["t"])
        assert sum(added) == g["pairs"] - 1 and added[0] == g["pairs"] - 1, name
        assert mate[g["rstar"]] == -1 and mate[g["a0"]] == -1 and mate[h] == g["r0"], name
        size, omate = oracle_matching(g["n"], g["f"], g["t"], with_mate=True)
        assert size == g["pairs"], name
        assert_matching(g["n"], g["f"], g["t"], omate, size)
    depth = colouring(n, f, t)
    assert (depth[[g["hub"] for _, g in parts]] == 0).all() and (depth[[g["a0"] for _, g in parts]] == 2).all()
    assert oracle_matching(n, f, t) == sum(g["pairs"] for _, g in parts)


def test_staircase_and_stars_round_by_round():
    for k in STAIRS:
        n, f, t = staircase(k)
        mate, added = greedy(n, f, t)
        assert added == [1] * min(k, GREEDY_ROUNDS), k
        assert (mate[:min(k, GREEDY_ROUNDS)] == k + np.arange(min(k, GREEDY_ROUNDS))).all(), k
        assert oracle_matching(n, f, t) == k
        # one round more would pair L_4 - R_4: the cap alone keeps it for the phases
        assert k <= GREEDY_ROUNDS or (mate[GREEDY_ROUNDS] == -1 and mate[k + GREEDY_ROUNDS] == -1)
    n, f, t = stars()
    mate, added = greedy(n, f, t)
    assert added == [len(STAR_SIZES), 0]
    assert oracle_matching(n, f, t) == len(STAR_SIZES) and int((colouring(n, f, t) % 2 == 0).sum()) == sum(STAR_SIZES)


def test_paths_leave_one_augmenting_path_each():
    cases = [(2 * k + 2, *path_edges(path_ids(k)), [path_ids(k)]) for k in PATHS]
    cases += [scattered_paths([3000], seed=1), scattered_paths(SCATTERED, seed=2)]
    for n, f, t, paths in cases:
        assert sorted(np.concatenate(paths).tolist()) == list(range(n))
        mate, added = greedy(n, f, t)
        depth = colouring(n, f, t)
        for ids in paths:
            k = len(ids) // 2 - 1
            assert (depth[ids[0::2]] % 2 == 0).all() and ids.min() == ids[-2]
            assert (mate[ids[2::2]] == ids[1:-1:2]).all() and mate[ids[0]] == -1 and mate[ids[-1]] == -1, k
        assert added == [sum(len(p) // 2 - 1 for p in paths), 0]
        size, omate = oracle_matching(n, f, t, with_mate=True)
        assert size == len(paths) + sum(added)
        assert_matching(n, f, t, omate, size)
        assert_matching(n, f, t, path_mate(n, paths), size)


@pytest.mark.parametrize("case", [TWO_ROOTS, TWO_ENDS], ids=["two_roots", "two_ends"])
def test_competing_trees_by_hand(case):
    n, f, t = case["n"], np.array(case["f"]), np.array(case["t"])
    mate, added = greedy(n, f, t)
    assert mate.tolist() == case["greedy"] and sum(added) == case["initial"]
    size, _ = oracle_matching(n, f, t, with_mate=True)
    assert size == case["matched"]
    assert_matching(n, f, t, np.array(case["mate"]), size)


# ---- on the device ---------------------------------------------------------------------------------------------------

def run(mm, n, f, t):
    """check() (two resident runs, the one-shot call, the certificate, the oracle), then the mate itself.
    -> (mate, stats)."""
    stats = check(mm, n, f, t)
    with mm.BfsGraph(n, np.asarray(f, dtype=np.uint64), np.asarray(t, dtype=np.uint64)) as g:
        mate, _, again = mm.bipartite_matching_run(g)
    assert no_ms(again) == no_ms(stats)
    return mate, stats


@pytest.mark.gpu
@pytest.mark.parametrize("degree", WALK_DEGREES)
def test_phase_walks_the_hub_list_from_a_level_2_frontier(mm, degree):
    """r* is the only free neighbour a phase can reach, and only through H's list, walked from the level-2 frontier
    (order[1..2), so lo > 0) by a thread, a warp or a block.  A dropped entry leaves matched at pairs - 1 and one phase;
    a tree growing past its end reaches the leaves at level 3."""
    for name, p, c, o in gadget_specs(degree):
        g = hub_gadget(degree, p, c, o)
        mate, st = run(mm, g["n"], g["f"], g["t"])
        pairs = g["pairs"]
        assert (st["initial_matched"], st["matched"], st["phases"], st["max_levels"]) == (pairs - 1, pairs, 2, 2), name
        assert st["left_vertices"] == pairs, name
        assert mate[g["rstar"]] == g["hub"] and mate[g["a0"]] == g["r0"], name


@pytest.mark.gpu
def test_all_gadgets_in_one_graph(mm):
    """One forest with a root per gadget: phase 1's level-2 frontier holds every hub, thread, warp and block walks
    together, and every tree ends at its own r*."""
    n, f, t, parts = all_gadgets()
    mate, st = run(mm, n, f, t)
    pairs = sum(g["pairs"] for _, g in parts)
    assert (st["initial_matched"], st["matched"], st["phases"], st["max_levels"]) == (pairs - len(parts), pairs, 2, 2)
    assert (mate[[g["rstar"] for _, g in parts]] == [g["hub"] for _, g in parts]).all()


@pytest.mark.gpu
def test_device_built_gadgets_equal_host_built(mm):
    import torch
    n, f, t, _ = all_gadgets()
    d_f = torch.from_numpy(f.astype(np.int32)).cuda()
    d_t = torch.from_numpy(t.astype(np.int32)).cuda()
    torch.cuda.synchronize()  # the library reads them on its own stream
    with mm.BfsGraph.from_device(n, len(f), d_f.data_ptr(), d_t.data_ptr()) as dev, mm.BfsGraph(n, f, t) as host:
        a, b = mm.bipartite_matching_run(dev), mm.bipartite_matching_run(host)
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    assert no_ms(a[2]) == no_ms(b[2]) and a[2]["matched"] == oracle_matching(n, f, t)


@pytest.mark.gpu
@pytest.mark.parametrize("k", STAIRS)
def test_greedy_rounds_stop_at_the_cap(mm, k):
    n, f, t = staircase(k)
    mate, st = run(mm, n, f, t)
    assert st["initial_matched"] == min(k, GREEDY_ROUNDS) and st["matched"] == k
    # past the cap, phase 1's trees each end at level 1 (R_j's pred is L_j); phase 2 has no root
    assert (st["phases"], st["max_levels"]) == ((1, 0) if k <= GREEDY_ROUNDS else (2, 1))
    assert (mate[:k] == k + np.arange(k)).all()


@pytest.mark.gpu
def test_greedy_rounds_stop_after_a_round_that_adds_nothing(mm):
    """Rounds 0 and 1 run and round 2 is not started; the cap would have run rounds 2 and 3 as well, which changes
    nothing but the work, so the work is what is asserted:
      entries  colouring: 2m each for the union-find, the forest and the same-level pass; round 0: every leaf (m);
               round 1: the free leaves (m - S); phase 1: the free leaves at level 1 (m - S), the first leaves at 2 (S)
      launches colouring 1 + 3 + 1 + 1 + 3 forest levels * 3 + 3 = 18; rounds 0 and 1: 6 each, and the free-L
               listing that stops round 2: 1; phase 1: 1 + 2 levels * 5 + the augment 1 = 12; the cover 1."""
    n, f, t = stars()
    m, s = len(f), len(STAR_SIZES)
    _, st = run(mm, n, f, t)
    assert (st["initial_matched"], st["matched"], st["phases"], st["max_levels"]) == (s, s, 1, 2)
    assert st["edges_inspected"] == 6 * m + m + 2 * (m - s) + s
    assert st["kernel_launches"] == 18 + 13 + 12 + 1


@pytest.mark.gpu
@pytest.mark.parametrize("k", PATHS)
def test_one_long_augmenting_path(mm, k):
    ids = path_ids(k)
    mate, st = run(mm, 2 * k + 2, *path_edges(ids))
    assert (st["initial_matched"], st["matched"], st["phases"], st["max_levels"]) == (k, k + 1, 2, k + 1)
    assert np.array_equal(mate, path_mate(2 * k + 2, [ids]))


@pytest.mark.gpu
@pytest.mark.parametrize("lengths,seed", [([3000], 1), (SCATTERED, 2)], ids=["one", "many"])
def test_scattered_augmenting_paths(mm, lengths, seed):
    """The flips walk scattered ids; with many paths, the trees end at their own levels, 2 .. 2501."""
    n, f, t, paths = scattered_paths(lengths, seed)
    mate, st = run(mm, n, f, t)
    k = sum(lengths)
    assert (st["initial_matched"], st["matched"], st["phases"], st["max_levels"]) == \
        (k, k + len(lengths), 2, max(lengths) + 1)
    assert np.array_equal(mate, path_mate(n, paths))


@pytest.mark.gpu
@pytest.mark.parametrize("case", [TWO_ROOTS, TWO_ENDS], ids=["two_roots", "two_ends"])
def test_competing_trees(mm, case):
    mate, st = run(mm, case["n"], case["f"], case["t"])
    assert mate.tolist() == case["mate"]
    assert [st[k] for k in ("initial_matched", "matched", "phases", "max_levels")] == \
        [case[k] for k in ("initial", "matched", "phases", "max_levels")]


# ---- one handle, every algorithm -------------------------------------------------------------------------------------

def handle_steps(n, f, t, w):
    """(name, graph -> outputs) of every algorithm on the BFS device graph, each called as its own tests call it."""
    from memgraph_b200 import betweenness as bcm
    from memgraph_b200 import connectivity as cc
    from memgraph_b200 import matching as mm

    def wsp(g):
        g.set_weights(f, t, w)
        return [g.weighted_distances(0, d, ub) for d, ub in [(OUT, None), (IN, None), (BOTH, None), (BOTH, 2)]]

    return [("matching", lambda g: [mm.bipartite_matching_run(g)]),
            ("bfs", lambda g: [g.distances(0, d) for d in (OUT, IN, BOTH)]),
            ("wcc", lambda g: [cc.wcc_run(g)]),
            ("biconnectivity", lambda g: [cc.biconnectivity_run(g, f, t)]),
            ("betweenness", lambda g: [bcm.bc_range(g, True, 0, 96), bcm.bc_range(g, False, 1000, 1064)]),
            ("wsp", wsp)]


def assert_same_run(a, b, what):
    for x, y in zip(a, b, strict=True):
        for u, v in zip(x, y, strict=True):
            if isinstance(u, dict):
                assert no_ms(u) == no_ms(v), what
            else:
                assert u.tobytes() == v.tobytes(), what


def assert_oracles(name, n, f, t, w, out):
    from _checkers import BfsOracle
    from test_bc_module import assert_matches
    from test_bc_oracle import oracle_bc
    from test_biconnectivity_oracle import oracle_biconnectivity
    from test_wcc_oracle import oracle_wcc
    from test_wsp_oracle import oracle_wsp, same_bits
    if name == "matching":
        mate, cover, st = out[0]
        certify(n, f, t, mate, cover, st)
        assert st["matched"] == oracle_matching(n, f, t)
    elif name == "bfs":
        oracle = BfsOracle()
        for d, (got, _) in zip((OUT, IN, BOTH), out):
            assert np.array_equal(got.astype(np.int64), oracle.distances(n, f, t, 0, d)), d
    elif name == "wcc":
        assert np.array_equal(out[0][0], oracle_wcc(n, f, t))
    elif name == "biconnectivity":
        bridge, bcc = oracle_biconnectivity(n, f, t)
        assert np.array_equal(out[0][0], bridge) and np.array_equal(out[0][1], bcc)
    elif name == "betweenness":
        assert_matches(out[0][0], oracle_bc(n, f, t, True, False, 0, 96))
        assert_matches(out[1][0], oracle_bc(n, f, t, False, False, 1000, 1064))
    else:
        for (d, ub), (dist, hops, _) in zip([(OUT, None), (IN, None), (BOTH, None), (BOTH, 2)], out):
            rc, ref, _, ref_hops, _ = oracle_wsp(n, f, t, w, 0, d, ub)
            assert rc == 0 and same_bits(dist, ref) and np.array_equal(hops, ref_hops), (d, ub)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["bipartite", "odd_cycles"])
def test_every_algorithm_on_one_handle(mm, kind):
    """Matching leaves the handle's depth array holding its colouring forest (bipartite or not) and its queues holding
    its searches; every algorithm after it, and matching after every other one, must answer as on a fresh handle."""
    import memgraph_b200 as mg
    from memgraph_b200 import bfs
    if kind == "bipartite":
        n, f, t = bipartite_rmat(14)
    else:
        n = 1 << 14
        f, t = mg.rmat_edges_host(14, 16 << 14)
    f, t = np.asarray(f, dtype=np.uint64), np.asarray(t, dtype=np.uint64)
    w = bfs.splitmix_weights(len(f))
    steps = handle_steps(n, f, t, w)
    fresh = {}
    for name, step in steps:
        with bfs.BfsGraph(n, f, t) as g:
            fresh[name] = step(g)
        assert_oracles(name, n, f, t, w, fresh[name])
    assert fresh["matching"][0][2]["bipartite"] == (kind == "bipartite")
    for order in (steps + steps[:1], steps[:1] + steps[:0:-1] + steps[:1]):
        with bfs.BfsGraph(n, f, t) as g:
            for i, (name, step) in enumerate(order):
                assert_same_run(step(g), fresh[name], (kind, i, name))

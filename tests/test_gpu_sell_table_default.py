"""-m gpu: the SELL walk's shared-memory table of the hottest labels, on by default on one partition.

With MGB200_SMEM_TABLE_KB unset, a one-partition handle takes the largest table the device gives the table kernel
(opt-in shared memory per block minus the kernel's static shared memory, in whole 16-byte TMA units) less 64 KB left to
L1, capped at n and rounded down to an even label count; several partitions keep the table opt-in.  A table slot holds
the same double as the contribution it copies and the add order inside a row does not change, so every algorithm that
gathers through the SELL walk -- PageRank, Katz, HITS and personalised PageRank -- must give the same bits with the
table as without it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
SCALE = 18  # 2^18 labels: the default table covers part of the gathered labels
PR = dict(max_iterations=20, stop_epsilon=0.0)
SEEDS = (np.array([0, 1, 2]), np.array([0.2, 0.5, 0.3]))


def optin_bytes():
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def rmat():
    import memgraph_b200 as mg
    n, m = 1 << SCALE, 16 << SCALE
    f, t = mg.rmat_edges_host(SCALE, m)
    return n, f, t


def three_vertices():
    return 3, np.array([0, 1, 2, 2], dtype=np.uint32), np.array([1, 2, 0, 1], dtype=np.uint32)


def katz_alpha(f, n):
    deg_max = np.bincount(np.asarray(f, dtype=np.int64), minlength=n).max()
    return float(0.9 / np.sqrt(deg_max + 1.0))


def table_labels(n, f, t, **kw):
    import memgraph_b200 as mg
    with mg.PageRankGraph.from_arrays(n, f, t, **kw) as g:
        return g.info["table_labels"]


def run_all(n, f, t):
    """Every algorithm that walks the SELL rows, on handles built under the current environment."""
    import memgraph_b200 as mg
    from memgraph_b200 import hits, katz
    from memgraph_b200 import personalized as P
    out = {}
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        out["table_labels"] = g.info["table_labels"]
        out["pagerank"] = g.run(**PR)[0]
        try:  # a guard, since the 3-vertex graph's ranking may never separate; both sides stop at the same iterate
            out["katz"] = katz.set_katz(g, alpha=katz_alpha(f, n), epsilon=1e-3, max_iterations=1000)[0]
        except katz.NotConverged as e:
            out["katz"] = e.centralities
        out["ppr_uniform"] = P.cugraph_pagerank(g)[0]
        out["ppr_seeded"] = P.cugraph_pagerank(g, personalization_vertices=SEEDS[0], personalization_values=SEEDS[1],
                                               max_iterations=100, stop_epsilon=1e-9)[0]
    with hits.HitsGraph(n, f, t) as h:
        out["hits_table_labels"] = tuple(i["table_labels"] for i in h.info)
        out["hubs"], out["authorities"], _ = h.run(max_iterations=20, tolerance=0.0)
    return out


def test_default_table_leaves_64k_of_the_largest_that_fits(monkeypatch):
    monkeypatch.delenv("MGB200_SMEM_TABLE_KB", raising=False)
    n, f, t = rmat()
    labels = table_labels(n, f, t)
    room = optin_bytes() - 65536  # what the default table leaves to L1 (core.hpp kTableL1Room)
    assert 0 < labels < n and labels % 2 == 0
    # the table and the kernel's mbarrier fit; no more than the static shared memory (128 bytes as compiled) and the
    # rounding to a 16-byte unit is left over
    assert 8 * labels + 8 <= room < 8 * labels + 128 + 16, (labels, room)


def test_an_explicit_size_may_take_the_largest_table(monkeypatch):
    monkeypatch.setenv("MGB200_SMEM_TABLE_KB", "100000")
    n, f, t = rmat()
    labels = table_labels(n, f, t)
    assert 8 * labels + 8 <= optin_bytes() < 8 * labels + 128 + 16, labels


@pytest.mark.parametrize("n", [1000, 1001, 3])
def test_default_table_is_capped_at_n_and_even(n, monkeypatch):
    monkeypatch.delenv("MGB200_SMEM_TABLE_KB", raising=False)
    rng = np.random.default_rng(n)
    f = rng.integers(0, n, 8 * n).astype(np.uint32)
    t = rng.integers(0, n, 8 * n).astype(np.uint32)
    assert table_labels(n, f, t) == n // 2 * 2


def test_zero_turns_the_table_off(monkeypatch):
    monkeypatch.setenv("MGB200_SMEM_TABLE_KB", "0")
    n, f, t = rmat()
    assert table_labels(n, f, t) == 0


def test_partitions_keep_the_table_opt_in(monkeypatch):
    import memgraph_b200 as mg
    monkeypatch.delenv("MGB200_SMEM_TABLE_KB", raising=False)
    n, f, t = rmat()
    for q in range(2):
        with mg.PageRankGraph.from_arrays(n, f, t, device=0, part_rank=q, part_world=2) as g:
            assert g.info["table_labels"] == 0


@pytest.mark.parametrize("graph", [rmat, three_vertices], ids=["rmat18", "n3"])
def test_table_gives_the_same_bits_as_the_plain_walk(graph, monkeypatch):
    n, f, t = graph()
    monkeypatch.delenv("MGB200_SMEM_TABLE_KB", raising=False)
    with_table = run_all(n, f, t)
    monkeypatch.setenv("MGB200_SMEM_TABLE_KB", "0")
    plain = run_all(n, f, t)
    assert 0 < with_table["table_labels"] <= n // 2 * 2
    assert all(x > 0 for x in with_table["hits_table_labels"])
    assert plain["table_labels"] == 0 and plain["hits_table_labels"] == (0, 0)
    for key in ["pagerank", "katz", "ppr_uniform", "ppr_seeded", "hubs", "authorities"]:
        assert np.array_equal(with_table[key], plain[key]), key


@pytest.mark.parametrize("mode", ["0", "1"], ids=["ticket", "static"])
def test_back_to_back_runs_on_one_handle_are_identical(mode, monkeypatch):
    """The ticket queue is rewound by the last CTA to leave; a second run that found it spent would skip every item."""
    import memgraph_b200 as mg
    monkeypatch.delenv("MGB200_SMEM_TABLE_KB", raising=False)
    monkeypatch.setenv("MGB200_SELL_MODE", mode)
    n, f, t = rmat()
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        assert g.info["table_labels"] > 0
        first = g.run(**PR)[0]
        second = g.run(**PR)[0]
    monkeypatch.setenv("MGB200_SMEM_TABLE_KB", "0")
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        plain = g.run(**PR)[0]
    assert np.array_equal(first, second)
    assert np.array_equal(first, plain)


def test_handles_with_different_tables_interleave(monkeypatch):
    """The table kernel's shared-memory limit belongs to the kernel, not to a handle: a handle with a smaller table
    that runs between two runs of one with a larger table must not leave the larger one unable to launch."""
    import memgraph_b200 as mg
    monkeypatch.delenv("MGB200_SMEM_TABLE_KB", raising=False)
    rng = np.random.default_rng(7)
    graphs = []
    for n in (2500, 2000):
        f = rng.integers(0, n, 8 * n).astype(np.uint32)
        t = rng.integers(0, n, 8 * n).astype(np.uint32)
        graphs.append(mg.PageRankGraph.from_arrays(n, f, t))
    large, small = graphs
    try:
        assert large.info["table_labels"] > small.info["table_labels"] > 0
        first = large.run(**PR)[0]
        small.run(**PR)
        assert np.array_equal(large.run(**PR)[0], first)
    finally:
        large.close()
        small.close()

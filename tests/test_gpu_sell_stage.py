"""-m gpu: SELL staging (graph_build.cu sell_staging, pagerank_kernels.cu cold_block_kernel / sell_walk).  A SELL entry whose
source lies in a block that has a pass is read from a value that pass staged, not from the gathered vector.  The
value is the same double and the add order inside a row is unchanged, so every algorithm that shares the gather must
give the same bits with staging on and off, count what scripts/block_model.py counts, and stage nothing where the
block class is off or the walk reads raw labels."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
from block_model import block_model  # noqa: E402

# small blocks, so that a small RMAT graph has several passes and SELL rows with sources in them; staging forced on, as by
# default it is on only where the gathered vector is larger than L2
ENV = {"MGB200_HEAVY_MIN_DEGREE": "64", "MGB200_BLOCK_FROM": "3000", "MGB200_BLOCK_LABELS": "2000", "MGB200_SELL_STAGE": "1"}
SCALE = 14


@pytest.fixture
def env(monkeypatch):
    for k, v in ENV.items():
        monkeypatch.setenv(k, v)
    return monkeypatch


def rmat(scale=SCALE):
    import memgraph_b200 as mg
    n, m = 1 << scale, 16 << scale
    return (n, *mg.rmat_edges_host(scale, m, seed=scale))


def model(n, f, t):
    e = os.environ
    return block_model(n, f, t, block_from=int(e["MGB200_BLOCK_FROM"]), block_labels=int(e["MGB200_BLOCK_LABELS"]),
                       heavy_min=int(e["MGB200_HEAVY_MIN_DEGREE"]), sell_blocks=0)


def everything(n, f, t):
    """PageRank (twice on one handle), Katz and personalised PageRank on one handle, then HITS on its own pair."""
    import memgraph_b200 as mg
    from memgraph_b200 import hits as H
    from memgraph_b200 import katz
    from memgraph_b200 import personalized as P
    out = {}
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        out["info"] = dict(g.info)
        out["pagerank"], _ = g.run(max_iterations=20, stop_epsilon=0.0)
        again, _ = g.run(max_iterations=20, stop_epsilon=0.0)
        assert np.array_equal(out["pagerank"], again)
        deg_max = int(np.bincount(np.asarray(f, dtype=np.int64), minlength=n).max())
        out["katz"], _ = katz.set_katz(g, alpha=0.9 / float(np.sqrt(deg_max + 1.0)), epsilon=1e-6)
        out["personalized"], _ = P.cugraph_pagerank(g, np.array([0, 17, 400]), np.array([0.2, 0.5, 0.3]),
                                                    max_iterations=20, stop_epsilon=0.0)
    with H.HitsGraph(n, f, t) as h:
        out["hits_info"] = h.info
        out["hubs"], out["authorities"], _ = h.run(max_iterations=30, tolerance=0.0)
    return out


def test_every_algorithm_is_bit_identical_with_staging_on_and_off(env):
    n, f, t = rmat()
    on = everything(n, f, t)
    env.setenv("MGB200_SELL_STAGE", "0")
    off = everything(n, f, t)
    want = model(n, f, t)
    assert on["info"]["blocks"] == want["blocks"] > 1
    assert on["info"]["stage_entries"] == want["stage_entries"] > 0
    assert all(side["stage_entries"] > 0 for side in on["hits_info"])
    assert off["info"]["stage_entries"] == 0 and all(side["stage_entries"] == 0 for side in off["hits_info"])
    for k in ("pagerank", "katz", "personalized", "hubs", "authorities"):
        assert np.array_equal(on[k], off[k]), k


def test_pad_entries_are_never_staged(env):
    """From label 0 on every source with in-SELL edges lies in a launched block: every real SELL entry is staged, and
    only the padding (slot n) is left."""
    import memgraph_b200 as mg
    env.setenv("MGB200_BLOCK_FROM", "0")
    env.setenv("MGB200_BLOCK_LABELS", "64")
    n, f, t = rmat(12)
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        info = dict(g.info)
    want = model(n, f, t)
    sell_edges = info["local_edges"] - info["heavy_edges"]
    assert info["stage_entries"] == want["stage_entries"]
    assert info["stage_entries"] <= sell_edges < info["sell_entries"]  # padding exists, and none of it is staged


def test_two_interleaved_handles_match_one_handle(env):
    import memgraph_b200 as mg
    n, f, t = rmat()
    n2, f2, t2 = rmat(13)
    with mg.PageRankGraph.from_arrays(n, f, t) as a, mg.PageRankGraph.from_arrays(n2, f2, t2) as b:
        assert a.info["stage_entries"] > 0 and b.info["stage_entries"] > 0
        ra1, _ = a.run(max_iterations=20, stop_epsilon=0.0)
        rb1, _ = b.run(max_iterations=20, stop_epsilon=0.0)
        ra2, _ = a.run(max_iterations=20, stop_epsilon=0.0)
        rb2, _ = b.run(max_iterations=20, stop_epsilon=0.0)
    with mg.PageRankGraph.from_arrays(n, f, t) as a:
        alone, _ = a.run(max_iterations=20, stop_epsilon=0.0)
    assert np.array_equal(ra1, ra2) and np.array_equal(rb1, rb2) and np.array_equal(ra1, alone)


@pytest.mark.parametrize("case", ["weighted", "lone_partition", "stream_kernel", "block_labels_0", "vector_fits_l2"])
def test_builds_without_staging_report_zero(env, case):
    import memgraph_b200 as mg
    from memgraph_b200 import personalized as P
    n, f, t = rmat(12)
    if case == "weighted":
        w = np.random.default_rng(6).uniform(0.5, 2.0, len(f))
        with P.weighted_graph(n, f, t, w) as g:
            assert g.info["stage_entries"] == 0
        return
    kw = {}
    if case == "lone_partition":
        env.setenv("MGB200_LONE_PARTITION", "1")
        kw = {"part_rank": 0, "part_world": 2}
    elif case == "stream_kernel":
        env.setenv("MGB200_SELL_KERNEL", "stream")
    elif case == "vector_fits_l2":  # the default: 4 K labels (32 KB) fit any L2
        env.delenv("MGB200_SELL_STAGE")
    else:
        env.setenv("MGB200_BLOCK_LABELS", "0")
    with mg.PageRankGraph.from_arrays(n, f, t, **kw) as g:
        assert g.info["stage_entries"] == 0
        if case in ("stream_kernel", "vector_fits_l2"):  # the block class itself stays on: only the staging is off
            assert g.info["blocks"] > 0

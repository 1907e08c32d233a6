"""-m gpu, one device: the vertex-partitioned PageRank path with every partition on device 0.

mgb200_graph_connect_peers accepts a peer on the same device (no peer access is needed), so P partitions built on
device 0 and run from P host threads exercise the whole partitioned path -- dealt and global labellings, the index
flags and the owner lookup, the shared-memory table whose slots ride in the flagged indices, need and push masks, the
flag-page barrier, the cross-partition rank sum, the collective abort and per-owner tiles -- on a machine with one GPU.

Every case runs in a child interpreter with three per-process settings:
- CUDA_DEVICE_MAX_CONNECTIONS=32: each partition drives 3 streams, and with more streams than hardware queues a
  spinning barrier kernel could sit in the same queue ahead of a peer's work and wait for it forever;
- CUDA_MODULE_LOADING=EAGER: under lazy loading, the first launch of a kernel may wait for the context to go idle,
  which it never does while another partition's barrier kernel spins on the same device waiting for this one (the
  barrier then times out on every partition);
- MGB200_BARRIER_TIMEOUT_MS=5000, so that a co-scheduling problem ends as an error in seconds."""
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from _checkers import Oracle

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REL_TOL = 1e-9
SCALE = 18  # 2^18 labels: L2_HOT_MB=1 (131072 / P labels per owner), L1_HOT_K=1 and a 1 KB table all end inside
            # every owner's label range, also at P = 8 (32768 labels per owner)
RUNS = [dict(max_iterations=20, damping_factor=0.85, stop_epsilon=0.0), dict()]  # fixed count, and the defaults
SMALL_TILES = {"MGB200_TILE_LABELS": "2048", "MGB200_TILE_HOT_MB": "1"}  # heavy rows gather tiled AND cold edges

# Variants that must not change a single bit of the result against the default run of the same P: they change how a
# gather learns its cache policy (index flags / owner lookup, L1 and L2 windows), the SELL kernel (hot table in shared
# memory: a TMA copy of the same contributions), how slices are handed to warps (every row is still summed by one lane
# in ascending source order), the epilogue's stream and grid, and where contributions are pushed (the gathered values
# are the same).  The rank sum is one fixed tree per partition and the partial sums are added in rank order everywhere.
EXACT = {
    "lookup": {"MGB200_IDX_FLAGS": "0"},
    "table1k": {"MGB200_SMEM_TABLE_KB": "1"},
    "table64k": {"MGB200_SMEM_TABLE_KB": "64"},
    "no_l1_hints": {"MGB200_L1_HOT_K": "-1"},
    "l1_1k": {"MGB200_L1_HOT_K": "1"},
    "l2_1mb": {"MGB200_L2_HOT_MB": "1"},
    # a table with an L1 window larger than the L2 window: code 01 of a flagged index must stay "table slot"
    "table1k_l2_0": {"MGB200_SMEM_TABLE_KB": "1", "MGB200_L2_HOT_MB": "0"},
    "table1k_l1_gt_l2": {"MGB200_SMEM_TABLE_KB": "1", "MGB200_L2_HOT_MB": "1", "MGB200_L1_HOT_K": "4096"},
    "ticket_small": {"MGB200_SELL_MODE": "0", "MGB200_SELL_WORK_ITEMS": "5"},
    "ticket_large": {"MGB200_SELL_MODE": "0", "MGB200_SELL_WORK_ITEMS": "100000"},
    "static_small": {"MGB200_SELL_MODE": "1", "MGB200_SELL_WORK_ITEMS": "5"},
    "static_large": {"MGB200_SELL_MODE": "1", "MGB200_SELL_WORK_ITEMS": "100000"},
    "no_overlap": {"MGB200_OVERLAP_EPILOGUE": "0"},
    "push_all_full_grid": {"MGB200_PUSH_MASK": "0", "MGB200_PUSH_CTAS": "0"},
    "push_all": {"MGB200_PUSH_MASK": "0", "MGB200_PUSH_CTAS": "2"},
    "push_mask_full_grid": {"MGB200_PUSH_MASK": "1", "MGB200_PUSH_CTAS": "0"},
}
# The same cache-policy variants over a layout with small per-owner tiles, where the heavy rows' cold edges go
# through the flags / lookup forms of the segment kernel (with the default tiles every heavy-row edge at this size is
# tiled).  Compared bit for bit with the default run of that layout.
EXACT_TILED = {
    "lookup": {"MGB200_IDX_FLAGS": "0"},
    "no_l1_hints": {"MGB200_L1_HOT_K": "-1"},
    "l1_1k": {"MGB200_L1_HOT_K": "1"},
    "l2_1mb": {"MGB200_L2_HOT_MB": "1"},
}
# Variants that relabel or regroup the sums, so only the tolerance applies: the global labelling gives other labels
# (so other ascending source orders inside a row), and tiles split a heavy row's sum into other partials.
TOLERANCE = {
    "global_labels": {"MGB200_LABELLING": "global"},
    "global_labels_push_all": {"MGB200_LABELLING": "global", "MGB200_PUSH_MASK": "0"},
    "small_tiles": SMALL_TILES,
}
WORLDS = [2, 3, 8]  # 3 deals an uneven split (2^18 % 3 = 1), 8 is the most partitions a graph may have


def in_child(fn, *args):
    """Run fn(*args) (a module-level function, JSON-able arguments) in a fresh interpreter; fail with its output."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys, json; sys.path[:0] = {[here, REPO]!r}; import {fn.__module__} as m; "
            f"m.{fn.__name__}(*json.loads({json.dumps(args)!r}))")
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32", CUDA_MODULE_LOADING="EAGER",
               MGB200_BARRIER_TIMEOUT_MS="5000")
    flags = ["-s"] if sys.flags.no_user_site else []
    proc = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=900, env=env)
    if proc.returncode:
        pytest.fail(proc.stdout + proc.stderr, pytrace=False)
    print(proc.stdout, end="")


def on_one_device(mg, n, f, t, world, **kw):
    from test_gpu_multi import run_partitioned
    got, results, infos = run_partitioned(mg, n, f, t, world, devices=[0] * world, **kw)
    its = {st.iterations for _, _, st in results}
    assert len(its) == 1, its  # every partition stops at the same iteration
    assert not np.isnan(got).any()
    assert sum(i["local_rows"] for i in infos) == n and sum(i["local_edges"] for i in infos) == len(f)
    return got, its.pop(), infos


def rel_err(got, ref):
    return float(np.max(np.abs(got - ref) / ref)) if len(ref) else 0.0


@pytest.fixture(scope="module")
def rmat_oracle(tmp_path_factory):
    """Oracle ranks and iteration counts of the RMAT graph for every entry of RUNS, in a file the children read."""
    import memgraph_b200 as mg
    n, m = 1 << SCALE, 16 << SCALE
    f, t = mg.rmat_edges_host(SCALE, m)
    oracle = Oracle()
    out = {}
    for i, kw in enumerate(RUNS):
        out[f"ranks{i}"], out[f"it{i}"] = oracle.pagerank(n, f, t, **kw)
    path = str(tmp_path_factory.mktemp("oracle") / f"rmat{SCALE}.npz")
    np.savez(path, **out)
    return path


def variant_case(world, layout, env, exact, ref_path):
    """Child: the default run of `layout` and the `env` variant of it, both against the oracle and, if `exact`, bit
    for bit against each other."""
    import memgraph_b200 as mg
    ref = np.load(ref_path)
    n, m = 1 << SCALE, 16 << SCALE
    f, t = mg.rmat_edges_host(SCALE, m)
    os.environ.update(layout)
    base = [on_one_device(mg, n, f, t, world, **kw) for kw in RUNS] if exact or not env else None
    os.environ.update(env)
    got = [on_one_device(mg, n, f, t, world, **kw) for kw in RUNS] if env else base
    for i, (ranks, it, infos) in enumerate(got):
        assert it == ref[f"it{i}"], (RUNS[i], it, int(ref[f"it{i}"]))
        err = rel_err(ranks, ref[f"ranks{i}"])
        assert err < REL_TOL, (RUNS[i], err)
        if exact and env:
            assert np.array_equal(ranks, base[i][0]), (RUNS[i], rel_err(ranks, base[i][0]))
        if layout.get("MGB200_TILE_HOT_MB") == "1" or env.get("MGB200_TILE_HOT_MB") == "1":
            for info in infos:  # every owner's heavy rows have tiled and cold edges
                assert 0 < info["tiled_edges"] < info["heavy_edges"], info
        print(f"P={world} {env} run {i}: iterations {it}, max rel err {err:.2e}")


@pytest.mark.parametrize("name", sorted(EXACT))
@pytest.mark.parametrize("world", WORLDS)
def test_variant_is_bit_identical(world, name, rmat_oracle):
    in_child(variant_case, world, {}, EXACT[name], True, rmat_oracle)


@pytest.mark.parametrize("name", sorted(EXACT_TILED))
@pytest.mark.parametrize("world", WORLDS)
def test_small_tiles_variant_is_bit_identical(world, name, rmat_oracle):
    in_child(variant_case, world, SMALL_TILES, EXACT_TILED[name], True, rmat_oracle)


@pytest.mark.parametrize("name", ["default"] + sorted(TOLERANCE))
@pytest.mark.parametrize("world", WORLDS)
def test_variant_meets_the_oracle(world, name, rmat_oracle):
    in_child(variant_case, world, {}, TOLERANCE.get(name, {}), False, rmat_oracle)


def _self_loops_and_multi_edges():
    rng = np.random.default_rng(11)
    n, m = 3000, 20000
    f, t = rng.integers(0, n, m), rng.integers(0, n, m)
    loops = rng.integers(0, n, 500)
    f = np.concatenate([f, loops, f[:3000], [5] * 2000])  # self-loops, 3000 repeated edges, and one edge
    t = np.concatenate([t, loops, t[:3000], [7] * 2000])  # repeated 2000 times (a heavy row)
    return n, np.stack([f, t], axis=1)


SMALL_GRAPHS = {  # name -> (partitions, n, edges)
    "n1_loop_P8": (8, 1, [[0, 0]]),  # one vertex: seven partitions own no row
    "n1_empty_P8": (8, 1, []),
    "n5_P8": (8, 5, [[0, 1], [1, 2], [2, 0], [3, 3], [4, 0], [4, 0]]),  # three partitions own no row
    "n5_empty_P8": (8, 5, []),
    "no_edges_P2": (2, 1000, []),  # every row is a zero row
    "self_loops_P3": (3, 7, [[1, 1], [1, 1], [2, 2]]),
    "loops_multi_P3": (3, *_self_loops_and_multi_edges()),
}


def small_graph_case(name):
    """Child: a small or degenerate graph against the oracle."""
    import memgraph_b200 as mg
    world, n, edges = SMALL_GRAPHS[name]
    e = np.array(edges, dtype=np.uint64).reshape(-1, 2)
    f, t = e[:, 0].copy(), e[:, 1].copy()
    for kw in RUNS:
        got, it, infos = on_one_device(mg, n, f, t, world, **kw)
        ref, rit = Oracle().pagerank(n, f, t, **kw)
        assert it == rit, (kw, it, rit)
        assert rel_err(got, ref) < REL_TOL, (kw, got, ref)
        assert abs(got.sum() - 1.0) < 1e-12
        print(f"P={world} n={n} m={len(f)} {kw}: rows per partition {[i['local_rows'] for i in infos]}")


@pytest.mark.parametrize("name", list(SMALL_GRAPHS))
def test_small_and_degenerate_graphs(name):
    in_child(small_graph_case, name)


def abort_case(world):
    """Child: one partition's host asks to abort -> every partition returns ERR_ABORTED (in the same iteration, so no
    barrier times out), and the same handles then run a normal call to the oracle's ranks."""
    import memgraph_b200 as mg
    from memgraph_b200 import _native as N
    scale = 16
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    graphs = [mg.PageRankGraph.from_arrays(n, f, t, device=0, part_rank=q, part_world=world) for q in range(world)]
    for g in graphs:
        g.connect_peers(local_graphs=graphs)
    outcome = [None] * world

    def work(q):
        try:  # stop_epsilon < 0 never converges: several 32-iteration batches until the abort
            outcome[q] = ("ok", graphs[q].run_partition(max_iterations=100000, stop_epsilon=-1.0,
                                                        should_abort=(lambda: True) if q == world - 1 else None))
        except mg.MgB200Error as e:
            outcome[q] = ("err", e.code, str(e))

    threads = [threading.Thread(target=work, args=(q,)) for q in range(world)]
    [th.start() for th in threads]
    [th.join(timeout=120) for th in threads]
    assert all(o is not None and o[0] == "err" and o[1] == N.ERR_ABORTED for o in outcome), outcome
    results = [None] * world

    def work2(q):
        results[q] = graphs[q].run_partition(max_iterations=20, stop_epsilon=0.0)

    threads = [threading.Thread(target=work2, args=(q,)) for q in range(world)]
    [th.start() for th in threads]
    [th.join(timeout=120) for th in threads]
    out = np.full(n, np.nan)
    for ranks, verts, st in results:
        assert st.iterations == 20
        out[verts.astype(np.int64)] = ranks
    for g in graphs:
        g.close()
    ref, _ = Oracle().pagerank(n, f, t, max_iterations=20, stop_epsilon=0.0)
    assert rel_err(out, ref) < REL_TOL


@pytest.mark.parametrize("world", [2, 3])
def test_abort_is_collective_and_handles_stay_usable(world):
    in_child(abort_case, world)


def single_partition_agreement_case():
    """Child: P = 2 on one device against the one-partition run of the same graph."""
    import memgraph_b200 as mg
    n, m = 1 << SCALE, 16 << SCALE
    f, t = mg.rmat_edges_host(SCALE, m)
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        single, st = g.run(max_iterations=20, stop_epsilon=0.0)
    multi, it, _ = on_one_device(mg, n, f, t, 2, max_iterations=20, stop_epsilon=0.0)
    err = rel_err(multi, single)
    print(f"P=2 on one device vs one partition: max relative difference {err:.3e}")
    assert st.iterations == it == 20
    assert err < 1e-12
    assert abs(multi.sum() - 1.0) < 1e-12


def test_two_partitions_match_one_partition():
    in_child(single_partition_agreement_case)

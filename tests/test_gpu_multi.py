"""-m gpu, needs >= 2 GPUs (skipped otherwise): the vertex-partitioned path.  Partitions live in ONE
process here (peer access between devices, one host thread per GPU, like the query module would drive
them); bench.py --gpus N exercises the one-process-per-GPU / CUDA-IPC variant of the same kernels."""
import threading

import numpy as np
import pytest

from _checkers import Oracle

pytestmark = pytest.mark.gpu
REL_TOL = 1e-9  # north_star: 1e-6


def _device_count():
    try:
        import memgraph_b200 as mg
        return mg.device_count()
    except Exception:
        return 0


def run_partitioned(mg, n, f, t, world, devices=None, **kw):
    """Partition q on device devices[q] (default: device q), one host thread each; -> (ranks by vertex, per-partition
    (ranks, vertices, RunStats), per-partition info)."""
    devices = list(range(world)) if devices is None else devices
    graphs = [mg.PageRankGraph.from_arrays(n, f, t, device=devices[q], part_rank=q, part_world=world)
              for q in range(world)]
    for g in graphs:
        g.connect_peers(local_graphs=graphs)
    results = [None] * world
    errors = []

    def work(q):
        try:
            results[q] = graphs[q].run_partition(**kw)
        except Exception as e:  # pragma: no cover
            errors.append((q, e))

    threads = [threading.Thread(target=work, args=(q,)) for q in range(world)]
    [th.start() for th in threads]
    [th.join() for th in threads]
    infos = [dict(g.info) for g in graphs]
    for g in graphs:
        g.close()
    assert not errors, errors
    out = np.full(n, np.nan)
    for ranks, verts, _ in results:
        out[verts.astype(np.int64)] = ranks
    return out, results, infos


@pytest.mark.parametrize("labelling,push_mask,push_ctas", [("dealt", "1", "2"), ("dealt", "0", "2"), ("dealt", "1", "0"),
                                                            ("global", "0", "2"), ("global", "1", "1")])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_partitioned_equals_oracle(world, labelling, push_mask, push_ctas, monkeypatch):
    if _device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    monkeypatch.setenv("MGB200_LABELLING", labelling)  # csrc/core.hpp RowMap: contiguous dealt ranges / global order
    monkeypatch.setenv("MGB200_PUSH_MASK", push_mask)  # 1: contributions go only to the partitions that gather them
    monkeypatch.setenv("MGB200_PUSH_CTAS", push_ctas)  # CTAs per SM of the push kernel next to the heavy-row kernel (0: full grid)
    import memgraph_b200 as mg
    oracle = Oracle()
    scale = 16
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    for kw in [dict(max_iterations=20, damping_factor=0.85, stop_epsilon=0.0), dict()]:
        got, results, infos = run_partitioned(mg, n, f, t, world, **kw)
        ref, it = oracle.pagerank(n, f, t, **kw)
        assert not np.isnan(got).any()
        assert all(st.iterations == it for _, _, st in results)  # every partition stops at the same iteration
        assert float(np.max(np.abs(got - ref) / ref)) < REL_TOL
        assert sum(i["local_rows"] for i in infos) == n and sum(i["local_edges"] for i in infos) == m
        edges = [i["local_edges"] for i in infos]
        assert max(edges) < 1.25 * (m / world) + 70000  # dealt round-robin by degree rank: edge-balanced
        assert all(i["heavy_rows"] + i["sell_rows"] + i["zero_rows"] == i["local_rows"] for i in infos)


def test_partitioned_matches_single_gpu_bitwise_sum():
    if _device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import os
    import memgraph_b200 as mg
    scale = int(os.environ.get("MGB200_MULTI_TEST_SCALE", "18"))
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        single, st1 = g.run(max_iterations=20, stop_epsilon=0.0)
    multi, results, _ = run_partitioned(mg, n, f, t, 2, max_iterations=20, stop_epsilon=0.0)
    err = float(np.max(np.abs(multi - single) / single))
    print(f"scale-{scale}: 2-GPU vs 1-GPU max relative difference {err:.3e}")
    assert err < 1e-12
    assert abs(multi.sum() - 1.0) < 1e-12


def test_one_call_multi_gpu_and_module_env(monkeypatch):
    """mgb200_parallel_iterative_pagerank_multi (host threads inside the call) and the module's MGB200_GPUS."""
    if _device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import memgraph_b200 as mg
    import _fakehost as fh
    from test_module_host import scattered_graph, oracle_through_module_semantics
    oracle = Oracle()
    n, m = 20_000, 150_000
    rng = np.random.default_rng(3)
    f, t = rng.integers(0, n, m), rng.integers(0, n, m)
    got, it = mg.pagerank_from_edges(n, f, t, max_iterations=30, stop_epsilon=0.0, gpus=2)
    ref, rit = oracle.pagerank(n, f, t, max_iterations=30, stop_epsilon=0.0)
    assert it == rit and float(np.max(np.abs(got - ref) / ref)) < REL_TOL
    monkeypatch.setenv("MGB200_GPUS", "2")
    gids, src, dst = scattered_graph(5000, 40000, seed=9)
    with fh.Module(fh.MODULE_SO) as module, fh.Graph(gids, src, dst) as g:
        nodes, ranks = module.call(g, 25, 0.85, 0.0, 1)
    order, exp, _ = oracle_through_module_semantics(oracle, gids, src, dst, max_iterations=25, stop_epsilon=0.0)
    assert np.array_equal(nodes, order) and float(np.max(np.abs(ranks - exp) / exp)) < REL_TOL


def test_abort_is_collective_and_handles_stay_usable():
    """ADVICE r1: one partition's host asks to abort -> EVERY partition leaves the loop in the same iteration with
    MGB200_ERR_ABORTED (no partition waits for a peer that already returned), and the same handles then run a normal
    call to the correct result (barrier counters still in step)."""
    if _device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import memgraph_b200 as mg
    from memgraph_b200 import _native as N
    scale, world = 16, 2
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    graphs = [mg.PageRankGraph.from_arrays(n, f, t, device=q, part_rank=q, part_world=world) for q in range(world)]
    for g in graphs:
        g.connect_peers(local_graphs=graphs)
    outcome = [None] * world

    def work(q, abort):
        try:
            # enough iterations for several 32-iteration batches; stop_epsilon < 0 never converges
            outcome[q] = ("ok", graphs[q].run_partition(max_iterations=100000, stop_epsilon=-1.0,
                                                        should_abort=(lambda: True) if abort else None))
        except mg.MgB200Error as e:
            outcome[q] = ("err", e)

    threads = [threading.Thread(target=work, args=(q, q == 1)) for q in range(world)]
    [th.start() for th in threads]
    [th.join(timeout=120) for th in threads]
    assert all(o is not None and o[0] == "err" and o[1].code == N.ERR_ABORTED for o in outcome), outcome
    # same handles, normal run
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
    assert float(np.max(np.abs(out - ref) / ref)) < REL_TOL


def test_partitions_built_from_the_generator_stream(monkeypatch):
    """mgb200_graph_create_rmat: every partition walks the generator a chunk at a time and keeps only its own edges
    (no device holds the whole COO).  Same ranks as the oracle on the materialised graph."""
    world = 2
    if _device_count() < world:
        pytest.skip("needs 2 GPUs")
    monkeypatch.setenv("MGB200_BUILD_CHUNK_EDGES", "50000")
    import memgraph_b200 as mg
    scale = 16
    n, m = 1 << scale, 16 << scale
    graphs = [mg.PageRankGraph.from_rmat(scale, m, device=q, part_rank=q, part_world=world) for q in range(world)]
    for g in graphs:
        g.connect_peers(local_graphs=graphs)
    results = [None] * world
    def work(q):
        results[q] = graphs[q].run_partition(max_iterations=20, stop_epsilon=0.0)
    threads = [threading.Thread(target=work, args=(q,)) for q in range(world)]
    [th.start() for th in threads]
    [th.join(timeout=120) for th in threads]
    out = np.full(n, np.nan)
    for ranks, verts, st in results:
        out[verts.astype(np.int64)] = ranks
    assert sum(g.info["local_edges"] for g in graphs) == m
    for g in graphs:
        g.close()
    f, t = mg.rmat_edges_host(scale, m)
    ref, _ = Oracle().pagerank(n, f, t, max_iterations=20, stop_epsilon=0.0)
    assert float(np.max(np.abs(out - ref) / ref)) < REL_TOL

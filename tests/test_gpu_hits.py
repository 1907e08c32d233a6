"""-m gpu: HITS hubs and authorities on the device (memgraph_b200/csrc/hits.cu) against the plain-C restatement
oracle/cugraph_hits_oracle.c, which is pinned on the reference's own cuGraph HITS e2e fixtures (test_hits_oracle.py).

Both directions of the graph are PageRank layouts, so the layout knobs and every gather variant apply to each; the
reductions have a fixed order, so a variant must give the default run's output bit for bit."""
import numpy as np
import pytest

from test_gpu_gather_variants import LAYOUT, VARIANTS
from test_hits_oracle import FIXTURES, check_fixture, fixture_arrays, oracle_hits

pytestmark = pytest.mark.gpu


def close(got, ref):
    return np.allclose(got, ref, rtol=1e-9, atol=1e-12)


def check_against_oracle(n, f, t, hubs, auth, st, **kw):
    ref_h, ref_a, it, conv = oracle_hits(n, f, t, **kw)
    assert (st["iterations"], bool(st["converged"])) == (it, conv), (st, it, conv)
    assert close(hubs, ref_h), float(np.max(np.abs(hubs - ref_h)))
    assert close(auth, ref_a), float(np.max(np.abs(auth - ref_a)))


@pytest.mark.parametrize("fx", FIXTURES, ids=lambda f: f["name"])
def test_reference_e2e_fixtures_on_the_device(fx):
    from memgraph_b200 import hits as H
    dense, f, t = fixture_arrays(fx)
    max_iterations, tolerance, normalized = fx["args"]
    kw = dict(max_iterations=max_iterations, tolerance=tolerance, normalized=normalized)
    with H.HitsGraph(len(dense), f, t) as g:
        hubs, auth, st = g.run(**kw)
    check_against_oracle(len(dense), f, t, hubs, auth, st, **kw)
    assert st["converged"]
    if fx["nodes"]:
        check_fixture(fx, hubs, auth, dense)
    one_h, one_a, one_st = H.hits(len(dense), f, t, **kw)  # the one-shot entry point
    assert np.array_equal(one_h, hubs) and np.array_equal(one_a, auth) and one_st["iterations"] == st["iterations"]


def random_multigraph(seed, n, m):
    """Multi-edges, self-loops, pure sources (no in-edge), pure sinks (no out-edge) and isolated vertices."""
    rng = np.random.default_rng(seed)
    hot = rng.integers(0, n, 8)  # a few heavy rows in both directions
    f = np.concatenate([rng.integers(0, n, m), hot.repeat(60), rng.integers(0, n, 480)])
    t = np.concatenate([rng.integers(0, n, m), rng.integers(0, n, 480), hot.repeat(60)])
    f[:40] = t[:40]  # self-loops
    f = np.concatenate([f, f[:200], np.full(30, n - 1)])  # multi-edges; vertex n - 1 is a pure source
    t = np.concatenate([t, t[:200], rng.integers(0, n - 3, 30)])
    t[t == n - 1] = 2
    sink = (f == n - 2)
    f[sink] = 0  # vertex n - 2 keeps its in-edges only: a pure sink
    f[(f == n - 3) | (t == n - 3)] = 0  # vertex n - 3 loses every edge: isolated
    t[t == n - 3] = 1
    return f, t


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_multigraphs(seed, monkeypatch):
    from memgraph_b200 import hits as H
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "16")
    n = [300, 2000, 5000][seed - 1]
    f, t = random_multigraph(seed, n, 8 * n)
    with H.HitsGraph(n, f, t) as g:
        fwd, rev = g.info
        assert fwd["heavy_rows"] > 0 and rev["heavy_rows"] > 0 and fwd["sell_rows"] > 0 and rev["sell_rows"] > 0
        for kw in [dict(), dict(normalized=False), dict(max_iterations=3, tolerance=0.0),
                   dict(max_iterations=0, tolerance=0.0), dict(max_iterations=500, tolerance=1e-13),
                   dict(max_iterations=500, tolerance=1e-13, normalized=False)]:
            hubs, auth, st = g.run(**kw)
            check_against_oracle(n, f, t, hubs, auth, st, **kw)
            if kw.get("normalized", True):
                assert abs(hubs.sum() - 1.0) < 1e-12 and abs(auth.sum() - 1.0) < 1e-12
            else:
                assert hubs.max() == 1.0 and auth.max() == 1.0
            assert hubs[n - 3] == 0.0 and auth[n - 3] == 0.0  # isolated
            assert auth[n - 1] == 0.0 and hubs[n - 2] == 0.0  # pure source, pure sink
        _, _, st = g.run(max_iterations=3, tolerance=0.0)
        assert st["iterations"] == 3 and not st["converged"]
        _, _, st = g.run(max_iterations=0, tolerance=0.0)
        assert st["iterations"] == 1 and not st["converged"]


SCALE = 18
RUN = dict(max_iterations=20, tolerance=0.0)


def rmat(scale):
    import memgraph_b200 as mg
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    return n, f, t


def run_rmat(env, monkeypatch):
    from memgraph_b200 import hits as H
    for k, v in {**LAYOUT, **env}.items():
        monkeypatch.setenv(k, v)
    n, f, t = rmat(SCALE)
    with H.HitsGraph(n, f, t) as g:
        first = g.run(**RUN)
        again = g.run(**RUN)
        info = g.info
    for a, b in zip(first[:2], again[:2]):
        assert np.array_equal(a, b)  # a second run on the same handle repeats every bit
    return first, info


@pytest.fixture(scope="module")
def baseline():
    with pytest.MonkeyPatch.context() as mp:
        return run_rmat({}, mp)


def test_rmat_layout_and_oracle(baseline):
    (hubs, auth, st), info = baseline
    for side in info:  # both handles carry every row class and tiled edges
        assert side["heavy_rows"] > 0 and side["sell_rows"] > 0 and side["zero_rows"] > 0, side
        assert 0 < side["tiled_edges"] < side["heavy_edges"], side
    n, f, t = rmat(SCALE)
    check_against_oracle(n, f, t, hubs, auth, st, **RUN)


def test_block_class_on_both_handles(baseline, monkeypatch):
    (hubs, auth, _), _ = baseline
    (bh, ba, st), info = run_rmat({"MGB200_BLOCK_FROM": "32768", "MGB200_BLOCK_LABELS": "16384"}, monkeypatch)
    for side in info:
        assert side["blocks"] > 1 and side["block_edges"] > 0, side
    assert close(bh, hubs) and close(ba, auth)
    n, f, t = rmat(SCALE)
    check_against_oracle(n, f, t, bh, ba, st, **RUN)


@pytest.mark.parametrize("name", list(VARIANTS))
def test_gather_variant_is_bit_identical(name, baseline, monkeypatch):
    (hubs, auth, st), _ = baseline
    (vh, va, vst), _ = run_rmat(VARIANTS[name], monkeypatch)
    assert vst["iterations"] == st["iterations"]
    assert np.array_equal(vh, hubs), float(np.max(np.abs(vh - hubs)))
    assert np.array_equal(va, auth), float(np.max(np.abs(va - auth)))


def test_graphs_without_edges():
    from memgraph_b200 import hits as H
    with H.HitsGraph(7, [], []) as g:
        hubs, auth, st = g.run()
        assert hubs.tolist() == [0.0] * 7 and auth.tolist() == [0.0] * 7
        assert st["iterations"] == 0 and st["converged"]
    hubs, auth, st = H.hits(0, [], [])
    assert len(hubs) == 0 and st["iterations"] == 0 and st["converged"]


def test_bad_endpoint_is_refused():
    from memgraph_b200 import hits as H
    from memgraph_b200.pagerank import MgB200Error
    with pytest.raises(MgB200Error, match="edge endpoint out of range"):
        H.HitsGraph(3, [0, 1], [1, 3])


def test_rmat_scale_20_against_the_oracle():
    from memgraph_b200 import hits as H
    n, f, t = rmat(20)
    kw = dict(max_iterations=30, tolerance=1e-6)
    with H.HitsGraph(n, f, t) as g:
        hubs, auth, st = g.run(**kw)
    check_against_oracle(n, f, t, hubs, auth, st, **kw)

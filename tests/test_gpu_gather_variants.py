"""-m gpu: every algorithm that gathers through launch_gather_phase's kernels -- PageRank, Katz, personalised PageRank and
weighted personalised PageRank -- under every gather variant, on one partition.

The graph is RMAT scale-18 with MGB200_HEAVY_MIN_DEGREE=64 and MGB200_TILE_HOT_MB=1, so that every boundary a gather
tests lies inside it: the default L1 window (16 K labels), the L2_HOT_MB=1 window and the tiled prefix (131072 labels
each), every table size below, and heavy rows with both tiled and cold edges next to SELL rows and zero rows.

A variant changes how a gather learns its cache policy, which kernel walks the SELL slices, how slices are handed to
warps, or whether the hottest labels are read from a shared-memory copy; none changes which values are summed or in
which order, so every result must equal the default run's bit for bit."""
import numpy as np
import pytest

from _checkers import Oracle
from test_cugraph_oracle import oracle_cugraph_pagerank
from test_katz_oracle import oracle_katz

pytestmark = pytest.mark.gpu
SCALE = 18
LAYOUT = {"MGB200_HEAVY_MIN_DEGREE": "64", "MGB200_TILE_HOT_MB": "1"}
PR = dict(max_iterations=20, stop_epsilon=0.0)
SEEDS = (np.array([0, 12345, 99999, 262143]), np.array([0.2, 0.5, 0.3, 1.0]))
PPR = {"uniform": dict(), "seeded": dict(personalization_vertices=SEEDS[0], personalization_values=SEEDS[1],
                                          max_iterations=100, stop_epsilon=1e-9)}

VARIANTS = {
    "flags": {"MGB200_IDX_FLAGS": "1"},
    "lookup": {"MGB200_IDX_FLAGS": "0", "MGB200_FORCE_MULTI_PATH": "1"},
    "multi_path": {"MGB200_FORCE_MULTI_PATH": "1"},
    "no_l1_hints": {"MGB200_L1_HOT_K": "-1"},
    "l1_1k": {"MGB200_L1_HOT_K": "1"},
    "l2_1mb": {"MGB200_L2_HOT_MB": "1"},
    "l2_0": {"MGB200_L2_HOT_MB": "0"},  # no evict-last span: every gather evict_first
    "l2_0_flags": {"MGB200_L2_HOT_MB": "0", "MGB200_IDX_FLAGS": "1"},
    "stream_kernel": {"MGB200_SELL_KERNEL": "stream"},
    "ticket_37": {"MGB200_SELL_MODE": "0", "MGB200_SELL_WORK_ITEMS": "37"},
    "static_5": {"MGB200_SELL_MODE": "1", "MGB200_SELL_WORK_ITEMS": "5"},
    "ticket_100000": {"MGB200_SELL_MODE": "0", "MGB200_SELL_WORK_ITEMS": "100000"},
    "no_overlap": {"MGB200_OVERLAP_EPILOGUE": "0"},
    "table0": {"MGB200_SMEM_TABLE_KB": "0"},
    "table1k": {"MGB200_SMEM_TABLE_KB": "1"},
    "table64k": {"MGB200_SMEM_TABLE_KB": "64"},
    "table200k": {"MGB200_SMEM_TABLE_KB": "200"},
    "table96k_flags": {"MGB200_SMEM_TABLE_KB": "96", "MGB200_IDX_FLAGS": "1"},
}


def close(got, ref):
    return float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-3))) < 1e-9


def dyadic_weights(m, seed=4):
    """Multiples of 1/4 below 4: every out-weight sum is exact in FP64, whatever order the atomics add in, so the
    weighted runs are bit-reproducible across builds."""
    return np.random.default_rng(seed).integers(1, 16, m) / 4.0


def run_all(env, monkeypatch):
    """PageRank, Katz and both personalised PageRanks on one unweighted handle, then the personalised PageRanks on a
    weighted one, all built under LAYOUT + env."""
    import memgraph_b200 as mg
    from memgraph_b200 import katz
    from memgraph_b200 import personalized as P
    for k, v in {**LAYOUT, **env}.items():
        monkeypatch.setenv(k, v)
    n, m = 1 << SCALE, 16 << SCALE
    f, t = mg.rmat_edges_host(SCALE, m)
    out = {}
    with mg.PageRankGraph.from_arrays(n, f, t) as g:
        out["info"] = dict(g.info)
        out["pagerank"] = g.run(**PR)
        out["katz"] = katz.set_katz(g, alpha=katz_alpha(f, n), epsilon=1e-3)
        for name, kw in PPR.items():
            out[f"ppr_{name}"] = P.cugraph_pagerank(g, **kw)
    with P.weighted_graph(n, f, t, dyadic_weights(m)) as g:
        for name, kw in PPR.items():
            out[f"wppr_{name}"] = P.cugraph_pagerank(g, **kw)
    return out


def katz_alpha(f, n):
    deg_max = np.bincount(np.asarray(f, dtype=np.int64), minlength=n).max()
    return float(0.9 / np.sqrt(deg_max + 1.0))  # alpha^2 deg_max < 1: gamma > 0, a real separation problem


@pytest.fixture(scope="module")
def baseline():
    with pytest.MonkeyPatch.context() as mp:
        return run_all({}, mp)


@pytest.fixture(scope="module")
def references():
    import memgraph_b200 as mg
    n, m = 1 << SCALE, 16 << SCALE
    f, t = mg.rmat_edges_host(SCALE, m)
    refs = {"pagerank": Oracle().pagerank(n, f, t, **PR)}
    rc, ranks, it = oracle_katz(n, f, t, katz_alpha(f, n), 1e-3)
    assert rc == 0
    refs["katz"] = (ranks, it)
    w = dyadic_weights(m)
    for name, kw in PPR.items():
        pers = (kw["personalization_vertices"], kw["personalization_values"]) if "personalization_vertices" in kw else None
        args = dict(personalization=pers, epsilon=kw.get("stop_epsilon", 1e-5), max_iterations=kw.get("max_iterations", 100))
        refs[f"ppr_{name}"] = oracle_cugraph_pagerank(n, f, t, **args)[:2]
        refs[f"wppr_{name}"] = oracle_cugraph_pagerank(n, f, t, weights=w, **args)[:2]
    return refs


def test_layout_puts_every_boundary_inside_the_graph(baseline):
    info = baseline["info"]
    assert info["heavy_rows"] > 0 and info["sell_rows"] > 0 and info["zero_rows"] > 0
    assert 0 < info["tiled_edges"] < info["heavy_edges"]  # heavy rows gather tiled and cold edges
    _, st = baseline["katz"]
    assert st["gamma"] > 0 and st["iterations"] >= 2


def check_against_references(out, refs):
    ranks, st = out["pagerank"]
    ref, it = refs["pagerank"]
    assert st.iterations == it == 20
    assert float(np.max(np.abs(ranks - ref) / ref)) < 1e-9
    cent, kst = out["katz"]
    ref, it = refs["katz"]
    assert kst["iterations"] == it and np.array_equal(cent, ref)  # Katz keeps the reference's rounding: bit-exact
    for key in ["ppr_uniform", "ppr_seeded", "wppr_uniform", "wppr_seeded"]:
        got, pst = out[key]
        ref, it = refs[key]
        assert pst["iterations"] == it, key
        assert close(got, ref), key


def test_default_run_meets_the_references(baseline, references):
    check_against_references(baseline, references)


@pytest.mark.parametrize("name", list(VARIANTS))
def test_variant_is_bit_identical_for_every_algorithm(name, baseline, references, monkeypatch):
    out = run_all(VARIANTS[name], monkeypatch)
    for key in ["pagerank", "katz", "ppr_uniform", "ppr_seeded", "wppr_uniform", "wppr_seeded"]:
        got, st = out[key]
        want, st0 = baseline[key]
        assert np.array_equal(got, want), (key, float(np.max(np.abs(got - want))))
    check_against_references(out, references)

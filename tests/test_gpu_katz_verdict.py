"""-m gpu: Katz centrality's convergence verdict on the device (memgraph_b200/csrc/katz.cu) against the oracle
(oracle/katz_oracle.cpp, pinned bit-exact to the reference's katz.cpp), where the verdict is hard:
  1. groups of equal centralities whose verdict depends on std::partial_sort's tie order, settled by the device's
     one-thread replay (katz_heap.hpp) -- small cases, the same with heavy rows and with shuffled vertex ids,
     mid-size random graphs and one tie gadget among 2^17 vertices;
  2. gamma = +inf (alpha^2 deg_max == 1 exactly) with epsilon <= 0, where vertices without in-edges have a NaN bound;
  3. negative alpha (centralities of both signs reach the descending radix sort) and alpha = 0;
  4. walk counts past 2^53, against an exact rational reference;
  5. other handles: weighted, reused after a guard-stopped run, and partitioned (refused).
Every device run carries an iteration guard: an input that fails to separate ends as NotConverged, never as a hang.
tests/test_katz_verdict_model.py restates the device's verdict in numpy; here it predicts `tie_order_runs`."""
import json
import math
from fractions import Fraction

import numpy as np
import pytest

from test_katz_verdict_model import (EPSILONS, GUARD, NON_FINITE_GAMMA, TIE_CASES, katz_model, oracle, permuted)

pytestmark = pytest.mark.gpu


def device(n, f, t, alpha, eps, guard=GUARD, graph=None):
    """-> (converged, centralities, stats) of one guarded device run (on `graph` if given, else a fresh handle)."""
    import memgraph_b200 as mg
    from memgraph_b200 import katz
    f = np.asarray(f, dtype=np.uint64)
    t = np.asarray(t, dtype=np.uint64)
    try:
        if graph is not None:
            c, st = katz.set_katz(graph, alpha, eps, guard)
        else:
            with mg.PageRankGraph.from_arrays(n, f, t) as g:
                c, st = katz.set_katz(g, alpha, eps, guard)
        return True, c, st
    except katz.NotConverged as e:
        return False, e.centralities, e.stats


def same_as_oracle(n, f, t, alpha, eps, guard=GUARD):
    """Device and oracle agree on the outcome, the iteration count and every bit of c."""
    want = oracle(n, f, t, alpha, eps, guard)
    got = device(n, f, t, alpha, eps, guard)
    assert got[0] == want[0], (got[0], want[0])
    assert got[2]["iterations"] == want[2], (got[2]["iterations"], want[2])
    assert np.array_equal(got[1], want[1]), float(np.max(np.abs(got[1] - want[1])))
    return got


# ---- 1. tie-order replays ---------------------------------------------------------------------------------------------

def check_replays(n, f, t, alpha, eps, expect_replay=True):
    model = katz_model(n, f, t, alpha, eps)
    converged, c, st = same_as_oracle(n, f, t, alpha, eps)
    assert converged
    assert st["tie_order_runs"] == len(model[3]), (st["tie_order_runs"], model[3])
    if expect_replay:
        assert st["tie_order_runs"] >= 1
    return model[3], st


@pytest.mark.parametrize("name", sorted(TIE_CASES))
def test_small_tie_replay(name):
    n, f, t, alpha, eps, replays, iterations = TIE_CASES[name]
    got, st = check_replays(n, f, t, alpha, eps)
    assert got == replays and st["iterations"] == iterations


@pytest.mark.parametrize("name", sorted(TIE_CASES))
def test_small_tie_replay_on_heavy_rows(name, monkeypatch):
    """Every row with two or more in-edges is a heavy row: the tied centralities come from katz_heavy_finish_kernel."""
    import memgraph_b200 as mg
    monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "2")
    n, f, t, alpha, eps, replays, iterations = TIE_CASES[name]
    with mg.PageRankGraph.from_arrays(n, np.asarray(f, dtype=np.uint64), np.asarray(t, dtype=np.uint64)) as g:
        assert g.info["heavy_rows"] > 0
    got, st = check_replays(n, f, t, alpha, eps)
    assert got == replays and st["iterations"] == iterations


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("name", sorted(TIE_CASES))
def test_small_tie_replay_with_shuffled_ids(name, seed):
    """Shuffled ids change partial_sort's input order and the device's labels; the model recomputes the outcome."""
    n, f, t, alpha, eps = permuted(TIE_CASES[name], seed)
    check_replays(n, f, t, alpha, eps, expect_replay=False)


def mid_case(seed):
    """A sparse random multigraph with n in 100..700, m ~ n, alpha = 2^-ceil(log2(deg_max + 1) / 2), eps = 2^-k."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(100, 701))
    m = int(rng.integers(n - n // 8, n + n // 8 + 1))
    f, t = rng.integers(0, n, m), rng.integers(0, n, m)
    deg_max = int(np.bincount(f, minlength=n).max())
    alpha = 2.0 ** -math.ceil(math.log2(deg_max + 1) / 2)
    eps = 2.0 ** -int(rng.integers(1, 9))
    return n, f, t, alpha, eps


# seeds of mid_case that reach a replay (14 of seeds 0..399), and whether it stopped the loop
MID_SEEDS = {4: False, 10: True, 22: False, 119: False, 167: False, 196: False, 262: True, 298: True, 303: True,
             336: True, 349: True, 382: False, 388: True, 399: True}


@pytest.mark.parametrize("seed", sorted(MID_SEEDS))
def test_mid_size_tie_replay(seed):
    replays, _ = check_replays(*mid_case(seed))
    assert replays[-1] == MID_SEEDS[seed]


def gadget_case(n=1 << 17, seed=5):
    """The stopping small case at scattered ids among n vertices; every other vertex is isolated (c = 0, ur = 0, so it
    passes the test every iteration).  The one-thread replay walks all n vertices."""
    gn, gf, gt = TIE_CASES["stops_n11"][:3]
    alpha, eps = TIE_CASES["stops_n11"][3:5]
    ids = np.random.default_rng(seed).choice(n, gn, replace=False)
    return n, ids[np.asarray(gf)], ids[np.asarray(gt)], alpha, eps


def test_large_tie_replay():
    n, f, t, alpha, eps = gadget_case()
    replays, st = check_replays(n, f, t, alpha, eps)
    print(f"2^17-vertex tie gadget: replays {replays}, iterations {st['iterations']}, "
          f"iterate_ms {st['iterate_ms']:.1f}")


def test_replays_ran_both_ways():
    """Each replay case above asserts its own outcome, so both outcomes occur on the device: some replay stopped the
    loop and some kept it going, in the small and in the mid-size cases."""
    small = [TIE_CASES[k][5][-1] for k in TIE_CASES]
    assert True in small and False in small
    assert True in MID_SEEDS.values() and False in MID_SEEDS.values()


# ---- 2. gamma = +inf and epsilon <= 0 ---------------------------------------------------------------------------------

@pytest.mark.parametrize("eps", EPSILONS)
@pytest.mark.parametrize("name", sorted(NON_FINITE_GAMMA))
def test_non_finite_gamma_and_non_positive_epsilon(name, eps):
    n, f, t, alpha = NON_FINITE_GAMMA[name]
    converged, c, st = same_as_oracle(n, f, t, alpha, eps)
    deg_max = np.bincount(f).max()
    assert st["max_out_degree"] == deg_max
    with np.errstate(divide="ignore"):
        gamma = np.float64(deg_max) / (1. - (alpha * alpha * np.float64(deg_max)))
    assert np.array_equal(np.float64(st["gamma"]), gamma), (st["gamma"], gamma)


# ---- 3. negative alpha and alpha = 0 ---------------------------------------------------------------------------------

def _random(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(200, 3000))
    m = int(n * rng.integers(2, 5))
    return n, rng.integers(0, n, m), rng.integers(0, n, m)


@pytest.mark.parametrize("kind", ["sqrt", "dyadic", "zero"])
@pytest.mark.parametrize("graph", ["random0", "random2", "rmat12"])
def test_negative_and_zero_alpha(graph, kind, monkeypatch):
    import memgraph_b200 as mg
    if graph == "rmat12":
        monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", "64")
        n = 1 << 12
        f, t = mg.rmat_edges_host(12, 8 << 12, seed=9)
    else:
        n, f, t = _random(int(graph[-1]))
    deg_max = int(np.bincount(np.asarray(f, dtype=np.int64), minlength=n).max())
    alpha = {"sqrt": -0.5 / math.sqrt(deg_max + 1.0),
             "dyadic": -(2.0 ** -math.ceil(math.log2(deg_max + 1) / 2)),
             "zero": 0.0}[kind]
    converged, c, st = same_as_oracle(n, f, t, alpha, 1e-3)
    assert converged
    if kind == "zero":
        assert not c.any() and st["iterations"] == 1
    else:
        assert (c > 0).any() and (c < 0).any()  # both signs went through the descending radix sort


# ---- 4. walk counts past 2^53 ----------------------------------------------------------------------------------------

def exact_katz(n, f, t, alpha, iterations):
    """Exact c_i = sum_{j <= i} alpha^j omega_j (Fractions) and omega_i (Python ints) for every i in `iterations`,
    and the largest walk count met on the way."""
    a = Fraction(alpha)
    omega = [1] * n
    edges = list(zip(np.asarray(f, dtype=np.int64).tolist(), np.asarray(t, dtype=np.int64).tolist()))
    scaled = [0] * n  # c_i * 2^(k i) with alpha = p / 2^k: scaled_i = scaled_(i-1) * 2^k + p^i omega_i
    p, q = a.numerator, a.denominator
    out, biggest = {}, 0
    for i in range(1, max(iterations) + 1):
        w = [0] * n
        for u, v in edges:
            w[v] += omega[u]
        omega = w
        biggest = max(biggest, max(omega))
        pi = p ** i
        scaled = [s * q + pi * o for s, o in zip(scaled, omega)]
        if i in iterations:
            out[i] = ([Fraction(s, q ** i) for s in scaled], list(omega))
    return out, biggest


def max_rel_err(got, exact):
    worst = 0.0
    for g, e in zip(got.tolist(), exact):
        if e == 0:
            assert g == 0.0
            continue
        worst = max(worst, float(abs(Fraction(g) - e) / abs(e)))
    return worst


def deciding_margin(state, alpha, gamma, eps, i):
    """How far the test `ur[b] - eps >= c[a]` over neighbours in c-descending order is from flipping at iteration i,
    relative to max |c|: the worst passing pair if it passed, the largest failing pair if it failed."""
    c_exact, omega = state
    c = np.array([float(x) for x in c_exact])
    ur = c + np.array([float(Fraction(alpha) ** (i + 1) * o) for o in omega]) * gamma
    order = np.argsort(-c, kind="stable")
    d = ur[order[1:]] - eps - c[order[:-1]]
    return abs(float(d.max())) / float(np.abs(c).max())


PAST_2_53 = {  # name -> (graph, seed, alpha, heavy-row threshold or None); every case has a deciding margin > 1e-9
    "random4000_s0": ("random", 0, 0.28125, None),
    "random4000_s1": ("random", 1, 0.28125, None),
    "random4000_s2": ("random", 2, 0.28125, None),
    "rmat14_heavy": ("rmat", 3, 2.0 ** -8, "64"),
}


@pytest.mark.parametrize("name", sorted(PAST_2_53))
def test_walk_counts_past_2_53(name, monkeypatch):
    import memgraph_b200 as mg
    kind, seed, alpha, heavy = PAST_2_53[name]
    eps = 1e-6
    if kind == "rmat":
        n = 1 << 14
        f, t = mg.rmat_edges_host(14, 4 << 14, seed=seed)
    else:
        rng = np.random.default_rng(seed)
        n = 4000
        f, t = rng.integers(0, n, 3 * n), rng.integers(0, n, 3 * n)
    if heavy:
        monkeypatch.setenv("MGB200_HEAVY_MIN_DEGREE", heavy)
        with mg.PageRankGraph.from_arrays(n, np.asarray(f, dtype=np.uint64), np.asarray(t, dtype=np.uint64)) as g:
            assert g.info["heavy_rows"] > 0 and g.info["tiled_edges"] > 0, g.info
    want = oracle(n, f, t, alpha, eps, guard=1000)
    got = device(n, f, t, alpha, eps, guard=1000)
    assert want[0] and got[0]
    it_o, it_d = want[2], got[2]["iterations"]
    exact, biggest = exact_katz(n, f, t, alpha, {it_o, it_d, it_o - 1})
    assert biggest > 2 ** 53
    err_o = max_rel_err(want[1], exact[it_o][0])
    err_d = max_rel_err(got[1], exact[it_d][0])
    assert err_o < 1e-12 and err_d < 1e-12, (err_o, err_d)
    deg_max = np.float64(np.bincount(np.asarray(f, dtype=np.int64), minlength=n).max())
    gamma = float(deg_max / (1. - alpha * alpha * deg_max))
    margin = min(deciding_margin(exact[it_o], alpha, gamma, eps, it_o),
                 deciding_margin(exact[it_o - 1], alpha, gamma, eps, it_o - 1))
    decisive = margin > 1e-9
    assert decisive, margin  # so the rounding past 2^53 cannot flip a verdict: the counts must be equal
    assert it_d == it_o
    print(name, json.dumps(dict(largest_walk_count_log2=round(math.log2(biggest), 1), iterations=it_d,
                                device_rel_err=err_d, oracle_rel_err=err_o, margin=margin,
                                bit_equal=bool(np.array_equal(got[1], want[1])))))


# ---- 5. handles --------------------------------------------------------------------------------------------------------

def test_weighted_handle_ignores_the_weights():
    from memgraph_b200 import personalized as P
    rng = np.random.default_rng(21)
    n = 1500
    f, t = rng.integers(0, n, 4 * n), rng.integers(0, n, 4 * n)
    deg_max = int(np.bincount(f, minlength=n).max())
    alpha = 0.5 / math.sqrt(deg_max + 1.0)
    want = oracle(n, f, t, alpha, 1e-3)
    with P.weighted_graph(n, f, t, rng.uniform(0.1, 3.0, len(f))) as g:
        assert g.info["tiled_edges"] == 0 and g.info["blocks"] == 0
        got = device(n, f, t, alpha, 1e-3, graph=g)
    assert want[0] and got[0] and got[2]["iterations"] == want[2]
    assert np.array_equal(got[1], want[1])


def test_guard_stopped_runs_leave_the_handle_reusable():
    """Guard 1, then guard 2 (the iteration that fills the zero in-degree rows' omega), then a full run on one handle:
    each equals the same run on a fresh handle, and the full run equals the oracle."""
    import memgraph_b200 as mg
    n, f, t, alpha, eps = mid_case(4)
    full = oracle(n, f, t, alpha, eps)
    assert full[0] and full[2] > 2
    with mg.PageRankGraph.from_arrays(n, np.asarray(f, dtype=np.uint64), np.asarray(t, dtype=np.uint64)) as g:
        assert g.info["zero_rows"] > 0
        for guard in (1, 2, GUARD):
            got = device(n, f, t, alpha, eps, guard=guard, graph=g)
            fresh = device(n, f, t, alpha, eps, guard=guard)
            assert got[0] == fresh[0] == (guard == GUARD)
            assert got[2]["iterations"] == fresh[2]["iterations"] == min(guard, full[2])
            assert np.array_equal(got[1], fresh[1])
    assert np.array_equal(got[1], full[1])


def partitioned_case():
    """Child: Katz on either partition of a two-partition graph on device 0 is refused, and those same handles then
    run partitioned PageRank to the oracle's ranks."""
    import threading
    import memgraph_b200 as mg
    from memgraph_b200 import katz
    from _checkers import Oracle
    rng = np.random.default_rng(8)
    n = 3000
    f, t = rng.integers(0, n, 20000), rng.integers(0, n, 20000)
    graphs = [mg.PageRankGraph.from_arrays(n, f, t, device=0, part_rank=q, part_world=2) for q in range(2)]
    for g in graphs:
        with pytest.raises(mg.MgB200Error, match=r"single partition \(part_world == 1\)"):
            katz.set_katz(g, 0.01, 1e-2, GUARD)
    for g in graphs:
        g.connect_peers(local_graphs=graphs)
    results = [None, None]

    def work(q):
        results[q] = graphs[q].run_partition(max_iterations=20, stop_epsilon=0.0)

    threads = [threading.Thread(target=work, args=(q,)) for q in range(2)]
    [th.start() for th in threads]
    [th.join() for th in threads]
    for g in graphs:
        g.close()
    got = np.full(n, np.nan)
    for ranks, verts, _ in results:
        got[verts.astype(np.int64)] = ranks
    ref, _ = Oracle().pagerank(n, f, t, max_iterations=20, stop_epsilon=0.0)
    assert float(np.max(np.abs(got - ref) / ref)) < 1e-9


def test_partitioned_handle_is_refused():
    from test_gpu_partitions_one_device import in_child
    in_child(partitioned_case)

"""A numpy restatement of memgraph_b200/csrc/katz.cu's iteration and convergence verdict, checked against the oracle
(oracle/katz_oracle.cpp, pinned bit-exact to the reference's katz.cpp).  No GPU needed.

The model does what the device does, step by step: the row epilogue with the reference's association, zero in-degree
rows that are never visited, the group analysis of the radix-sorted centralities (verdict_like_the_kernels) and, when a
group's verdict depends on std::partial_sort's tie order, the replay of that order (katz.tie_order, the host copy of the
device's katz_heap.hpp).  It also reports which iterations needed that replay, so that the GPU tests
(tests/test_gpu_katz_verdict.py) can predict the device's `tie_order_runs`.

Two families of inputs matter here:
  * gamma = +inf (alpha^2 * deg_max == 1 exactly, so the denominator is +0) with epsilon <= 0.  The reference computes ur = c + (alpha^(i+1) *
    omega) * gamma for every vertex, so a zero in-degree vertex has ur = 0 + (+-0 * inf) = NaN, which fails no
    comparison.  A device that kept ur = 0 for those rows would see `0 - eps >= 0` hold for each of them: two such
    vertices in the c = 0 group make the verdict "not converged" forever.  `zero_row_fix=False` models that device.
  * dyadic alpha on small graphs, where centralities are exact and ties are common: the rare groups whose verdict
    depends on partial_sort's tie order occur, both ways (the replay stops the loop, or keeps it going)."""
import math

import numpy as np
import pytest

from test_katz_oracle import oracle_katz
from test_katz_tie_order import verdict_like_the_kernels

GUARD = 64  # every run here is bounded: an input that never separates ends as "not converged", never as a hang


def katz_model(n, f, t, alpha, eps, guard=GUARD, zero_row_fix=True):
    """-> (converged, c[n], iterations, replays) where replays lists, for every iteration whose verdict needed the
    tie-order replay, True when the replay stopped the loop and False when it kept it going."""
    f = np.asarray(f, dtype=np.int64)
    t = np.asarray(t, dtype=np.int64)
    c = np.zeros(n)
    if len(f) == 0:
        return True, c, 0, []
    deg_max = np.float64(np.bincount(f, minlength=n).max())
    with np.errstate(divide="ignore"):
        gamma = float(deg_max / (1. - (alpha * alpha * deg_max)))  # +inf when alpha^2 * deg_max == 1
    zero_rows = np.bincount(t, minlength=n) == 0
    omega = np.ones(n)
    replays = []
    iteration = 0
    while True:
        iteration += 1
        # walk counts are integers: below 2^53 every summation order gives the same omega
        w = np.bincount(t, weights=omega[f], minlength=n)
        a_i = math.pow(alpha, float(iteration))
        a_next = math.pow(alpha, float(iteration + 1))
        c = c + a_i * w  # numpy rounds each operation once, like __dadd_rn / __dmul_rn
        with np.errstate(invalid="ignore"):
            ur = c + (a_next * w) * gamma  # 0 * inf = NaN where omega = 0 and gamma is not finite
        # rows nobody visits: c = 0, and ur = 0 + 0 * gamma (NaN when gamma is not finite) -- or 0 on the unfixed device
        c[zero_rows] = 0.0
        ur[zero_rows] = 0.0 + 0.0 * gamma if zero_row_fix else 0.0
        with np.errstate(invalid="ignore"):
            converged, ambiguous = verdict_like_the_kernels(c, ur, eps)
            replayed = ambiguous > 0 and not _definite_fail(c, ur, eps)
        if replayed:
            replays.append(bool(converged))
        omega = w
        if converged or iteration >= guard:
            return converged, c, iteration, replays


def _definite_fail(c, ur, eps):
    """katz.cu's `definite_fail`: the verdict is "not converged" under every order of equal centralities."""
    n = len(c)
    rows = np.argsort(-c, kind="stable")
    ks = c[rows]
    first = np.r_[True, ks[1:] != ks[:-1]]
    start = np.maximum.accumulate(np.where(first, np.arange(n), 0))
    bound = ur[rows] - eps
    if np.any((start > 0) & (bound >= ks[np.maximum(start - 1, 0)])):
        return True
    strict_per_group = np.bincount(start, weights=(bound >= ks).astype(np.float64), minlength=n)
    return bool(np.any(strict_per_group >= 2))


def oracle(n, f, t, alpha, eps, guard=GUARD):
    rc, c, it = oracle_katz(n, np.asarray(f, dtype=np.uint64), np.asarray(t, dtype=np.uint64), alpha, eps, guard)
    assert rc in (0, 3), rc
    return rc == 0, c, it


# ---- graphs where alpha^2 * deg_max == 1 exactly (gamma = +inf), and finite-gamma controls ----------------------------

def _graphs():
    out_star_dag = (8, [0, 0, 0, 0, 1, 5], [1, 2, 3, 4, 5, 6])  # the example: deg_max 4, two zero in-degree vertices
    return {
        # name: (n, f, t, alpha)
        "dag_deg4_a0.5": (*out_star_dag, 0.5),
        "dag_deg4_a-0.5": (*out_star_dag, -0.5),
        "dag_deg4_a0.25_control": (*out_star_dag, 0.25),
        "dag_deg16_a0.25": (20, [0] * 16 + [1, 2, 3], list(range(1, 17)) + [17, 18, 19], 0.25),
        "dag_deg16_a0.125_control": (20, [0] * 16 + [1, 2, 3], list(range(1, 17)) + [17, 18, 19], 0.125),
        "chain_a1": (6, [0, 1, 2, 3], [1, 2, 3, 4], 1.0),
        "chain_a0.5_control": (6, [0, 1, 2, 3], [1, 2, 3, 4], 0.5),
        # cycles: gamma = inf never separates, both sides run into the guard
        "cycle_deg4_a0.5": (7, [0, 0, 0, 0, 1, 2, 3, 4], [1, 2, 3, 4, 0, 0, 0, 0], 0.5),
        "ring_a1": (5, [0, 1, 2, 3, 4], [1, 2, 3, 4, 0], 1.0),
        # multi-edges and self-loops count towards deg_max: 2 + 1 + 1 = 4 out-edges at vertex 0
        "multi_loop_deg4_a-0.5": (6, [0, 0, 0, 0, 2, 3], [1, 1, 0, 2, 4, 5], -0.5),
        "multi_loop_deg4_a0.25_control": (6, [0, 0, 0, 0, 2, 3], [1, 1, 0, 2, 4, 5], 0.25),
    }


NON_FINITE_GAMMA = _graphs()
EPSILONS = [1e-2, 0.0, -1e-3]


@pytest.mark.parametrize("eps", EPSILONS)
@pytest.mark.parametrize("name", sorted(NON_FINITE_GAMMA))
def test_model_equals_the_oracle_at_non_finite_gamma(name, eps):
    n, f, t, alpha = NON_FINITE_GAMMA[name]
    deg_max = np.bincount(f).max()
    assert (alpha * alpha * deg_max == 1.0) == (not name.endswith("_control"))
    want = oracle(n, f, t, alpha, eps)
    got = katz_model(n, f, t, alpha, eps)
    assert got[0] == want[0] and got[2] == want[2], (got[0], got[2], want[0], want[2])
    assert np.array_equal(got[1], want[1])


@pytest.mark.parametrize("alpha,eps,iterations", [(0.5, 0.0, 3), (0.5, -1e-3, 3), (-0.5, 0.0, 2), (0.5, 1e-2, 3)])
def test_zero_in_degree_rows_decide_the_non_finite_gamma_verdict(alpha, eps, iterations):
    """n = 8, 0 -> {1, 2, 3, 4}, 1 -> 5 -> 6: deg_max 4, so alpha = +-0.5 gives gamma = +inf.  The oracle converges;
    the model converges with it, and without the zero-row fix it runs into the guard whenever eps <= 0."""
    n, f, t = 8, [0, 0, 0, 0, 1, 5], [1, 2, 3, 4, 5, 6]
    want = oracle(n, f, t, alpha, eps)
    assert want[0] and want[2] == iterations
    fixed = katz_model(n, f, t, alpha, eps)
    assert fixed[0] and fixed[2] == iterations and np.array_equal(fixed[1], want[1])
    unfixed = katz_model(n, f, t, alpha, eps, zero_row_fix=False)
    if eps <= 0:
        assert not unfixed[0] and unfixed[2] == GUARD
    else:
        assert unfixed[0] and unfixed[2] == iterations


# ---- tie-order replays -----------------------------------------------------------------------------------------------

# (n, f, t, alpha, eps, replay outcomes, iterations) -- found by a seeded search over small random multigraphs
TIE_CASES = {
    "stops_n11": (11, [0, 4, 2, 10, 2, 7], [6, 9, 1, 0, 9, 0], 0.5, 2.0 ** -5, [True], 2),
    "continues_n10": (10, [8, 0, 5, 6, 7, 3, 1], [3, 5, 3, 4, 0, 4, 3], 0.5, 0.25, [False], 3),
}


def permuted(case, seed):
    """The same graph with its vertex ids shuffled: partial_sort's input order and the device's labels change."""
    n, f, t = case[:3]
    perm = np.random.default_rng(seed).permutation(n)
    return n, perm[np.asarray(f)], perm[np.asarray(t)], *case[3:5]


@pytest.mark.parametrize("name", sorted(TIE_CASES))
def test_model_replays_ties_like_the_oracle(name):
    n, f, t, alpha, eps, replays, iterations = TIE_CASES[name]
    want = oracle(n, f, t, alpha, eps)
    got = katz_model(n, f, t, alpha, eps)
    assert got[0] and want[0]
    assert got[2] == want[2] == iterations
    assert np.array_equal(got[1], want[1])
    assert got[3] == replays
    for seed in range(8):
        pn, pf, pt, pa, pe = permuted(TIE_CASES[name], seed)
        want = oracle(pn, pf, pt, pa, pe)
        got = katz_model(pn, pf, pt, pa, pe)
        assert got[0] == want[0] and got[2] == want[2] and np.array_equal(got[1], want[1]), seed


def small_tie_search(draws, seed=2024):
    """Seeded draws of small multigraphs with dyadic alpha and epsilon: the model against the oracle on every draw."""
    rng = np.random.default_rng(seed)
    stopped = continued = 0
    for _ in range(draws):
        n = int(rng.integers(2, 13))
        m = int(rng.integers(1, 2 * n))
        f, t = rng.integers(0, n, m), rng.integers(0, n, m)
        alpha = float(rng.choice([0.5, 0.25, 0.125]))
        eps = float(2.0 ** -rng.integers(0, 7))
        want = oracle(n, f, t, alpha, eps)
        got = katz_model(n, f, t, alpha, eps)
        assert got[0] == want[0] and got[2] == want[2] and np.array_equal(got[1], want[1]), (n, f, t, alpha, eps)
        stopped += sum(got[3])
        continued += len(got[3]) - sum(got[3])
    return stopped, continued


def test_model_equals_the_oracle_on_random_small_graphs():
    stopped, continued = small_tie_search(3000)
    assert stopped >= 3 and continued >= 3, (stopped, continued)

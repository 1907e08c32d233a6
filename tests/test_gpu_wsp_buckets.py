"""Delta-stepping at every bucket width (memgraph_b200/csrc/wsp.cu, `MGB200_WSP_DELTA`).  The bucket width changes the
work of an unbounded run, never its result: every width, from 5e-324 to 1e300, must give totals byte-identical to the
default width and to oracle/wsp_oracle.c, with equal hops.  Each run also asserts the bucket count that the oracle's
totals imply, so a width that stops reaching the case it was chosen for (distances on bucket ends, `nextafter` bucket
ends, +inf totals in the far pile, one bucket) fails instead of passing quietly."""
import math

import numpy as np
import pytest

import memgraph_b200 as mg
from memgraph_b200 import bfs
from test_wsp_oracle import oracle_wsp, same_bits

pytestmark = pytest.mark.gpu

UNREACHED = 0x7FF0000000000001  # wsp.cu's kUnreached: above +inf
INF_BITS = 0x7FF0000000000000
SMALLEST = 5e-324


def bits(x):
    return int(np.float64(x).view(np.uint64))


def bucket_end(x_bits, delta):
    """wsp.cu's bucket_end on bit patterns: the end of the delta-wide bucket holding x, strictly above x."""
    if x_bits >= INF_BITS:
        return UNREACHED
    x = float(np.uint64(x_bits).view(np.float64))
    with np.errstate(over="ignore"):
        t = float((np.floor(np.float64(x) / np.float64(delta)) + 1.0) * np.float64(delta))
    if not t > x:
        t = math.nextafter(x, math.inf)
    return UNREACHED if math.isinf(t) else bits(t)


def expected_buckets(totals, delta):
    """The buckets an unbounded run processes, from its final totals.  When the near pile empties below threshold T, the
    smallest far distance is the smallest final total at or above T (its shortest path's last vertex below T has been
    relaxed with its final value), so the sequence of thresholds follows from the totals alone."""
    d = np.unique(np.asarray(totals, dtype=np.float64)[~np.isnan(totals)].view(np.uint64))
    t, count = bucket_end(0, delta), 1
    while True:
        i = int(np.searchsorted(d, np.uint64(t)))
        if t >= UNREACHED or i == len(d):
            return count
        t, count = bucket_end(int(d[i]), delta), count + 1


def splitmix_unit(m, salt):
    """Seeded uniforms in [0, 1) independent of bfs.splitmix_weights."""
    z = np.arange(1, m + 1, dtype=np.uint64) + np.uint64(salt) * np.uint64(0x632BE59BD9B4E019)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0**-53


def weights(kind, m):
    u = bfs.splitmix_weights(m)
    if kind == "uniform":
        return u
    if kind == "int":
        return bfs.splitmix_weights(m, "int")
    if kind == "log":  # log-uniform over 2^-30 .. 2^30
        return np.exp2(u * 60.0 - 30.0)
    if kind == "zeros":  # 30 % exact zeros among uniform weights
        w = u.copy()
        w[splitmix_unit(m, 1) < 0.3] = 0.0
        return w
    if kind == "huge":  # two hops overflow to +inf; the host-side weight sum overflows, so the default width is 1.0
        return 1e308 + u * 0.7e308
    if kind == "subnormal":  # multiples of the smallest subnormal: every sum is exact
        return bfs.splitmix_weights(m, "int") * SMALLEST
    raise ValueError(kind)


KINDS = ("uniform", "int", "log", "zeros", "huge", "subnormal")


def run(g, source, direction, delta, monkeypatch, upper_bound=None):
    if delta is None:
        monkeypatch.delenv("MGB200_WSP_DELTA", raising=False)
    else:
        monkeypatch.setenv("MGB200_WSP_DELTA", repr(float(delta)))
    try:
        return g.weighted_distances(source, direction, upper_bound)
    finally:
        monkeypatch.delenv("MGB200_WSP_DELTA", raising=False)


@pytest.fixture(scope="module")
def rmat14():
    scale = 14
    n, m = 1 << scale, 16 << scale
    f, t = mg.rmat_edges_host(scale, m)
    source = int(np.bincount(f.astype(np.int64), minlength=n).argmax())
    return n, f, t, source


@pytest.mark.parametrize("direction", [0, 1, 2])
@pytest.mark.parametrize("kind", KINDS)
def test_rmat_delta_sweep(rmat14, monkeypatch, kind, direction):
    n, f, t, source = rmat14
    w = weights(kind, len(f))
    rc, dist, _, hops, _ = oracle_wsp(n, f, t, w, source, direction)
    assert rc == 0
    finite = dist[np.isfinite(dist)]
    positive = finite[finite > 0]
    assert len(positive) > 1000, (kind, direction)
    typical = float(np.sort(positive)[len(positive) // 2])  # np.median would average two 1e308s into +inf
    with bfs.BfsGraph(n, f, t) as g:
        g.set_weights(f, t, w)
        base_d, base_h, base = run(g, source, direction, None, monkeypatch)
        assert same_bits(base_d, dist) and np.array_equal(base_h, hops), (kind, direction)
        if kind == "huge":
            assert base["delta"] == 1.0 and np.isinf(dist).any()
        assert base["buckets"] == expected_buckets(dist, base["delta"]), (kind, direction)
        # 2^-60 of the typical total: floor(x / delta) + 1 no longer moves past x, so bucket ends come from nextafter
        tiny = typical * 2.0**-60
        deltas = [1.0, 0.5] if kind == "int" else []
        deltas += [tiny] if tiny >= SMALLEST else []
        deltas += [SMALLEST, 1e300]
        for delta in deltas:
            ctx = (kind, direction, delta)
            gd, gh, st = run(g, source, direction, delta, monkeypatch)
            assert st["delta"] == delta, ctx
            assert gd.tobytes() == base_d.tobytes() and np.array_equal(gh, hops), ctx
            assert st["reached"] == base["reached"], ctx
            want = expected_buckets(dist, delta)
            assert st["buckets"] == want, ctx
            if delta == 1e300:
                # one bucket is Bellman-Ford; near-overflow totals start above 1e300 and keep a bucket each
                assert want == 1 if kind != "huge" else want > 100, ctx
            elif delta == SMALLEST and positive.min() >= 2.0**-50:
                # after the zero-total bucket, x / delta overflows: the threshold jumps straight to "unreached"
                assert want == 2, ctx
            elif delta in (1.0, 0.5):  # integer totals: every one sits on a bucket end
                assert want == 1 + len(np.unique(finite)), ctx
            elif delta == tiny:
                if kind == "int":  # one bucket per distinct total
                    assert want == 1 + len(np.unique(finite)), ctx
                else:
                    assert want >= 100, ctx
        # a bounded run has no buckets: the knob is ignored
        gd, gh, st = run(g, source, direction, 0.5, monkeypatch, upper_bound=3)
        rc, d3, _, h3, _ = oracle_wsp(n, f, t, w, source, direction, 3)
        assert rc == 0 and same_bits(gd, d3) and np.array_equal(gh, h3)
        assert st["delta"] == 0.0 and st["buckets"] == 0


def test_knob_values_that_are_ignored(monkeypatch):
    n = 6
    f, t = np.array([0, 1, 2, 3, 4]), np.array([1, 2, 3, 4, 5])
    w = np.array([1.0, 2.0, 3.0, 4.0, 5.0])
    with bfs.BfsGraph(n, f, t) as g:
        g.set_weights(f, t, w)
        base_d, base_h, base = run(g, 0, 0, None, monkeypatch)
        for text in ("0", "-1", "nan", "inf", "-inf", "abc", "", "1.5x", "1e999"):
            monkeypatch.setenv("MGB200_WSP_DELTA", text)
            d, h, st = g.weighted_distances(0)
            assert st["delta"] == base["delta"], text
            assert d.tobytes() == base_d.tobytes() and np.array_equal(h, base_h), text
        monkeypatch.setenv("MGB200_WSP_DELTA", "2.5")
        d, _, st = g.weighted_distances(0)
        assert st["delta"] == 2.5 and d.tobytes() == base_d.tobytes()
        # totals 1 3 6 10 15: the buckets [0, 2.5) [2.5, 5) [5, 7.5) [10, 12.5) [15, 17.5)
        assert st["buckets"] == expected_buckets(d, 2.5) == 5


def grid(side):
    """side x side grid, both directions of every edge."""
    v = np.arange(side * side).reshape(side, side)
    a = np.concatenate([v[:, :-1].ravel(), v[:-1, :].ravel()])
    b = np.concatenate([v[:, 1:].ravel(), v[1:, :].ravel()])
    return side * side, np.concatenate([a, b]), np.concatenate([b, a])


@pytest.mark.parametrize("kind", ["uniform", "int"])
def test_grid_many_buckets_with_large_far_piles(monkeypatch, kind):
    n, f, t = grid(256)
    w = weights(kind, len(f))
    with bfs.BfsGraph(n, f, t) as g:
        g.set_weights(f, t, w)
        for direction in (0, 2):
            rc, dist, _, hops, _ = oracle_wsp(n, f, t, w, 0, direction)
            assert rc == 0
            gd, gh, st = run(g, 0, direction, None, monkeypatch)
            ctx = (kind, direction)
            assert same_bits(gd, dist) and np.array_equal(gh, hops), ctx
            assert st["reached"] == n - 1, ctx
            assert st["buckets"] == expected_buckets(dist, st["delta"]) > 10, ctx

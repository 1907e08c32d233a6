#!/usr/bin/env python3
"""Strongly connected components measurement: prints one JSON line.

GPU arm, per workload: the graph built on the device, one warm-up run, then the median of --runs runs of
mgb200_scc_run.  Workloads: RMAT at each of --scales (the benchmark's generator, 16 edges per vertex, device-resident);
a DAG of cycles ("blocks" of 1 to 64 vertices, about 2^--dag-log vertices, block edges from lower to higher blocks,
ids shuffled); one cycle of 2^--cycle-log vertices in shuffled order.  Reported per workload:
  build_s                 wall time of making the edges and building the CSR + CSC on the device
  ms                      median CUDA-event time (first kernel .. last label written)
  edges_per_s             m / t
  hbm_bound_fraction      (LOWER_BOUND_BYTES / 3.35 TB/s) / t, where LOWER_BOUND_BYTES = 4 * edges_inspected (each
                          inspected adjacency entry is a 4-byte id) + 2 * 8 * n (out- and in-offsets read once to count)
                          + 4 * 4 * n (the two counts written, the representative written and read by the numbering)
                          + 8 * n (the labels written) -- a lower bound on the HBM time as a share of the time taken;
                          NOT a bandwidth reached
  stats                   the run's mgb200_scc_stats
  bfs_ms                  yardstick: one mgb200_bfs_run OUT from the same pivot (the live vertex with the largest
                          in * out product after the trim, recomputed here on the host), median CUDA-event time
  check                   the output against oracle/scc_oracle.c on the same edges in the same run (true / false), or
                          null with check_skipped saying why (not enough host memory for the uint64 COO and the oracle)
networkx arm: the wall time of networkx.strongly_connected_components on RMAT --nx-scale (a MultiDiGraph of every
vertex and edge, as the reference's nxalg builds it, construction excluded): a floor for nxalg's time, null where
networkx is not installed.  The card's name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the measurement still stands; the card is then reported unknown
        return {"name": None, "power_limit": None, "error": str(e)}


def available_host_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def lower_bound_bytes(n, stats):
    return 4 * stats["edges_inspected"] + 16 * n + 16 * n + 8 * n


def host_pivot(n, f, t):
    """The pivot scc.cu picks, from the host: full trim, then the largest in * out (ties: smaller id)."""
    keep = f != t
    f, t = f[keep].astype(np.int64), t[keep].astype(np.int64)
    live = np.ones(n, dtype=bool)
    while True:
        e = live[f] & live[t]
        ind = np.bincount(t[e], minlength=n)
        outd = np.bincount(f[e], minlength=n)
        drop = live & ((ind == 0) | (outd == 0))
        if not drop.any():
            break
        live &= ~drop
    key = np.where(live, ind.astype(np.uint64) * outd.astype(np.uint64), 0)
    return int(np.argmax(key)) if live.any() else None


def measure(g, n, m, runs, f, t, build_s, name):
    from memgraph_b200.connectivity import scc_run
    from test_scc_oracle import oracle_scc
    scc_run(g)  # warm-up: module load, allocations
    times, got, stats = [], None, None
    for _ in range(runs):
        got, stats = scc_run(g)
        times.append(stats["run_ms"])
    t_s = float(np.median(times)) / 1e3
    out = {"workload": name, "n": n, "m": m, "build_s": build_s, "ms": float(np.median(times)), "ms_all": times,
           "edges_per_s": m / t_s, "lower_bound_bytes": lower_bound_bytes(n, stats),
           "hbm_bound_fraction": lower_bound_bytes(n, stats) / HBM_BYTES_PER_S / t_s, "stats": stats}
    if f is None:
        out["check"] = None
        out["check_skipped"] = (f"host memory: {available_host_bytes() / 2**30:.1f} GiB available, the uint64 COO and "
                                f"the oracle need about {(24 * m + 48 * n) / 2**30:.1f} GiB")
        out["bfs_ms"] = None
        return out
    t0 = time.perf_counter()
    exp = oracle_scc(n, f, t)
    out["check"] = bool(np.array_equal(got, exp))
    out["oracle_s"] = time.perf_counter() - t0
    pivot = host_pivot(n, f, t)
    if pivot is not None:
        bfs = []
        for _ in range(runs + 1):
            _, st = g.distances(pivot)
            bfs.append(st["traverse_ms"])
        out["bfs_pivot"], out["bfs_ms"] = pivot, float(np.median(bfs[1:]))
    return out


def rmat_arm(scale, runs):
    import memgraph_b200 as mg
    from memgraph_b200 import _native as N
    from memgraph_b200.connectivity import BfsGraph
    lib = N.lib()
    n, m = 1 << scale, 16 << scale
    can_check = available_host_bytes() > 1.25 * (24 * m + 48 * n)
    d_from, d_to = N.vp(), N.vp()
    for p in (d_from, d_to):
        if lib.mgb200_device_malloc(0, m * 4, ctypes.byref(p)):
            raise RuntimeError(lib.mgb200_last_error().decode())
    f = t = None
    try:
        t0 = time.perf_counter()
        mg.rmat_edges_device(scale, m, d_from, d_to, seed=42, device=0)
        g = BfsGraph.from_device(n, m, d_from, d_to)
        build_s = time.perf_counter() - t0
        if can_check:
            f, t = np.empty(m, dtype=np.uint32), np.empty(m, dtype=np.uint32)
            for host, dev in ((f, d_from), (t, d_to)):
                if lib.mgb200_copy_to_host(0, host.ctypes.data, dev, m * 4):
                    raise RuntimeError(lib.mgb200_last_error().decode())
            f, t = f.astype(np.uint64), t.astype(np.uint64)
    finally:
        lib.mgb200_device_free(0, d_from)
        lib.mgb200_device_free(0, d_to)
    with g:
        return measure(g, n, m, runs, f, t, build_s, f"rmat_{scale}")


def host_arm(name, n, f, t, runs):
    from memgraph_b200.connectivity import BfsGraph
    t0 = time.perf_counter()
    g = BfsGraph(n, f, t)
    build_s = time.perf_counter() - t0
    with g:
        return measure(g, n, len(f), runs, f, t, build_s, name)


def block_dag(log_n, seed=5):
    rng = np.random.default_rng(seed)
    sizes = rng.integers(1, 65, (1 << log_n) // 32)
    blocks = len(sizes)
    start = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    n = int(sizes.sum())
    member = np.repeat(np.arange(blocks), sizes)
    ids = np.arange(n)
    nxt = ids + 1
    last = start + sizes - 1
    nxt[last] = start  # each block a cycle (a one-vertex block gets a self-loop, which changes nothing)
    a, b = rng.integers(0, blocks, 2 * blocks), rng.integers(0, blocks, 2 * blocks)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    keep = lo != hi
    bf = start[lo[keep]] + rng.integers(0, 64, keep.sum()) % sizes[lo[keep]]
    bt = start[hi[keep]] + rng.integers(0, 64, keep.sum()) % sizes[hi[keep]]
    perm = rng.permutation(n)
    del member
    return n, perm[np.concatenate([ids, bf])].astype(np.uint64), perm[np.concatenate([nxt, bt])].astype(np.uint64)


def networkx_arm(scale):
    try:
        import networkx as nx
    except ImportError:
        return None
    from _checkers import oracle_rmat_edges
    n = 1 << scale
    f, t = oracle_rmat_edges(scale)
    g = nx.MultiDiGraph()
    g.add_nodes_from(range(n))
    g.add_edges_from(zip(f.tolist(), t.tolist()))
    t0 = time.perf_counter()
    comps = list(nx.strongly_connected_components(g))
    return {"scale": scale, "n": n, "m": len(f), "networkx": nx.__version__, "s": time.perf_counter() - t0,
            "components": len(comps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="22,24")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--dag-log", type=int, default=22)
    ap.add_argument("--cycle-log", type=int, default=20)
    ap.add_argument("--nx-scale", type=int, default=16)
    args = ap.parse_args()
    result = {"workload": "strongly_connected_components", "card": card(), "gpu": []}
    for s in args.scales.split(","):
        result["gpu"].append(rmat_arm(int(s), args.runs))
    n, f, t = block_dag(args.dag_log)
    result["gpu"].append(host_arm(f"block_dag_{args.dag_log}", n, f, t, args.runs))
    n = 1 << args.cycle_log
    perm = np.random.default_rng(3).permutation(n).astype(np.uint64)
    result["gpu"].append(host_arm(f"cycle_{args.cycle_log}", n, perm, np.roll(perm, -1), args.runs))
    result["networkx"] = networkx_arm(args.nx_scale)
    print(json.dumps(result))


if __name__ == "__main__":
    main()

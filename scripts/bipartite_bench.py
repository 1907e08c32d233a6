#!/usr/bin/env python3
"""Maximum bipartite matching measurement: prints one JSON line.

GPU arm, per graph: the BFS device graph built from a host COO, one warm-up run, then the median of --runs runs of
mgb200_bipartite_matching_run.  The graphs:
  bipartite RMAT s   the benchmark's RMAT(s, 16 * 2^s edges, seed 42) with (u, v) -> (u, 2^s + v): skewed degrees on
                     both sides, 2 * 2^s vertices
  uniform s          16 * 2^s uniformly random edges between two sides of 2^s vertices each (seed 42)
  plain RMAT s       the RMAT graph itself, which has odd cycles: it times the colouring and the reject path
Reported per graph:
  build_s            wall time of building the CSR + CSC on the device from the host COO
  ms                 median CUDA-event time (first kernel .. last output, no transfers)
  stats              the run's mgb200_matching_stats (phases, max_levels, initial_matched, matched, edges_inspected)
  lower_bound_bytes  4 * edges_inspected (each inspected entry is a 4-byte id) + 16 * n (the out- and in-offsets read
                     at least once) -- a lower bound on the HBM traffic; hbm_bound_fraction is its time at 3.35 TB/s
                     over the time taken, NOT a bandwidth reached
  check / oracle_s   the answer against oracle/bipartite_oracle.c (colouring + Hopcroft-Karp) on the same edges, and
                     the oracle's wall time
CPU arm: one CALL of the reference's own module (oracle/_ref, built by build() where a reference checkout exists)
against ours on the fake mgp host (tests/mgp_wcc_host.cpp), bipartite RMAT at --cpu-scales, wall time each, in a child
interpreter on a thread with a 1 GiB stack (the reference's recursive DFS overflows 8 MB from scale 12 on); null where
oracle/_ref was not built.  The card's name and power limit are read in the same run.
"""
import argparse
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
REF_MODULE_SO = os.path.join(REPO, "oracle", "_ref", "bipartite_matching_reference.so")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the measurement still stands; the card is then reported unknown
        return {"name": None, "power_limit": None, "error": str(e)}


def graph(kind, scale):
    import memgraph_b200 as mg
    half, m = 1 << scale, 16 << scale
    if kind == "uniform":
        rng = np.random.default_rng(42)
        return 2 * half, rng.integers(0, half, m, dtype=np.uint64), half + rng.integers(0, half, m, dtype=np.uint64)
    f, t = mg.rmat_edges_host(scale, m, seed=42)
    return (2 * half, f, t + np.uint64(half)) if kind == "bipartite_rmat" else (half, f, t)


def gpu_arm(kind, scale, runs):
    from memgraph_b200.matching import BfsGraph, bipartite_matching_run
    from test_bipartite_oracle import oracle_matching
    n, f, t = graph(kind, scale)
    out = {"graph": kind, "scale": scale, "n": n, "m": len(f)}
    t0 = time.perf_counter()
    g = BfsGraph(n, f, t)
    out["build_s"] = time.perf_counter() - t0
    with g:
        bipartite_matching_run(g)  # warm-up: module load, allocations
        times, stats = [], None
        for _ in range(runs):
            _, _, stats = bipartite_matching_run(g)
            times.append(stats["run_ms"])
    t_s = float(np.median(times)) / 1e3
    lb = 4 * stats["edges_inspected"] + 16 * n
    out.update({"ms": float(np.median(times)), "ms_all": times, "lower_bound_bytes": lb,
                "hbm_bound_fraction": lb / HBM_BYTES_PER_S / t_s, "stats": stats})
    t0 = time.perf_counter()
    expected = oracle_matching(n, f, t)
    out["oracle_s"] = time.perf_counter() - t0
    out["oracle_matched"] = expected
    out["check"] = expected == stats["matched"]
    return out


CPU_ARM_CODE = """
import json, sys, threading, time
sys.path[:0] = [%(tests)r, %(repo)r]
import test_bipartite_module as bm
from test_bipartite_oracle import bipartite_rmat
out = []


def run():
    for scale in %(scales)r:
        n, f, t = bipartite_rmat(scale)
        row = {"scale": scale, "n": n, "m": len(f), "stack_bytes": 1 << 30}
        for name, path in (("reference", bm.REF_MODULE_SO), ("gpu_module", bm.MODULE_SO)):
            with bm.Module(path) as module:
                if name == "gpu_module":
                    bm.call(module, n, f, t)  # the device module's first call also initialises CUDA
                t0 = time.perf_counter()
                row[name] = bm.call(module, n, f, t)
                row[name + "_s"] = time.perf_counter() - t0
        row["speedup"] = row["reference_s"] / row["gpu_module_s"]
        row["equal"] = row["reference"] == row["gpu_module"]
        out.append(row)


threading.stack_size(1 << 30)
th = threading.Thread(target=run)
th.start()
th.join()
print(json.dumps(out))
"""


def cpu_arm(scales):
    if not os.path.exists(REF_MODULE_SO):
        return None
    code = CPU_ARM_CODE % {"tests": os.path.join(REPO, "tests"), "repo": REPO, "scales": scales}
    proc = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=3600)
    if proc.returncode:
        return {"error": (proc.stdout + proc.stderr)[-2000:]}
    return json.loads(proc.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bipartite-scales", default="20,22,24")
    ap.add_argument("--uniform-scales", default="20,22")
    ap.add_argument("--plain-scales", default="22")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--cpu-scales", default="12,14")
    args = ap.parse_args()
    scales = lambda s: [int(x) for x in s.split(",") if x]  # noqa: E731
    result = {"workload": "bipartite_matching", "card": card(), "gpu": []}
    for kind, arg in (("bipartite_rmat", args.bipartite_scales), ("uniform", args.uniform_scales),
                      ("plain_rmat", args.plain_scales)):
        for s in scales(arg):
            result["gpu"].append(gpu_arm(kind, s, args.runs))
            print(json.dumps(result["gpu"][-1]), file=sys.stderr, flush=True)  # progress; the result line is stdout
    result["cpu"] = cpu_arm(scales(args.cpu_scales))
    print(json.dumps(result))


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""HITS measurement: prints one JSON line per scale as soon as that scale is done (so an interrupted run keeps what it
finished), then one line with every scale together.

Per scale: an RMAT graph from the benchmark's generator (mg.rmat_edges_host, seed 42, 16 edges per vertex) built into a
memgraph_b200.hits.HitsGraph (forward + reverse PageRank layouts).  Reported:
  build_ms_forward / _reverse   device build time of each handle (mgb200_graph_info.build_ms)
  create_s                      wall time of HitsGraph() (upload + both builds + permutations)
  hits_ms_per_iteration         median over --runs runs of --iterations iterations at tolerance 0.0 (after one warm-up
                                run) of the run's CUDA-event time / iterations; the run includes the two output writes
  hits_edges_per_s              2 * m * iterations / time (each iteration gathers every edge twice)
  kernel_launches_per_iteration from the run's stats
  pagerank_ms_per_iteration     mgb200_pagerank_run on a PageRankGraph of the same COO in the same process, same run
                                count and iterations (stop_epsilon 0), iterate_ms / iterations
  ratio                         hits_ms_per_iteration / pagerank_ms_per_iteration
  max_rel_err                   against oracle/cugraph_hits_oracle.c on the same input and parameters (relative, with
                                a 1e-12 absolute floor), only where the host has the memory and scale <= --check-max-scale
A scale is skipped, with the reason, before anything is generated when its estimated peak does not fit: host memory
(HOST_BYTES_PER_EDGE) against MemAvailable, device memory (DEVICE_BYTES_PER_EDGE) against the card's total; a build
that still runs out of device memory is reported as skipped with the library's error.  The card's
name and power limit are read in the same run (a read-only query).
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

# host peak per edge: the uint64 COO (16), the uint32 copies made for the HITS handle (8) and the pinned staging
HOST_BYTES_PER_EDGE = 16 + 8 + 8
# device peak per edge, while the reverse handle is built: the uint32 COO (8), the forward layout (about 6) and the
# build's transients (about 40).  The PageRank handle is built after the HITS handle is gone.
DEVICE_BYTES_PER_EDGE = 8 + 6 + 40


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


def device_total_bytes():
    import ctypes
    from memgraph_b200 import _native as N
    name, sms, total = ctypes.create_string_buffer(256), ctypes.c_int(0), ctypes.c_size_t(0)
    if N.lib().mgb200_device_info(0, name, 256, ctypes.byref(sms), ctypes.byref(total)):
        raise RuntimeError(N.lib().mgb200_last_error().decode())
    return total.value


def progress(*what):
    print(*what, file=sys.stderr, flush=True)


def max_rel_err(got, ref):
    return float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-12))) if len(ref) else 0.0


def gpu_arm(scale, runs, iterations, check_max_scale):
    import memgraph_b200 as mg
    from memgraph_b200 import hits as H
    n, m = 1 << scale, 16 << scale
    need = HOST_BYTES_PER_EDGE * m + 64 * n
    device_need = DEVICE_BYTES_PER_EDGE * m + 256 * n
    out = {"scale": scale, "n": n, "m": m, "iterations": iterations}
    if available_host_bytes() < 1.1 * need:
        out["skipped"] = (f"host memory: {available_host_bytes() / 2**30:.1f} GiB available, the COO and its copies "
                          f"need about {need / 2**30:.1f} GiB")
        return out
    if device_total_bytes() < 1.05 * device_need:
        out["skipped"] = (f"device memory: {device_total_bytes() / 2**30:.1f} GiB on the card, two HITS layouts, a "
                          f"PageRank layout and the build need about {device_need / 2**30:.1f} GiB")
        return out
    f, t = mg.rmat_edges_host(scale, m, seed=42)
    kw = dict(max_iterations=iterations, tolerance=0.0, normalized=True)
    t0 = time.perf_counter()
    try:
        g = H.HitsGraph(n, f, t)
    except mg.MgB200Error as e:  # the estimate above was too low for this card
        out["skipped"] = f"HITS graph build failed: {e}"
        return out
    with g:
        out["create_s"] = time.perf_counter() - t0
        fwd, rev = g.info
        out["build_ms_forward"], out["build_ms_reverse"] = fwd["build_ms"], rev["build_ms"]
        out["resident_bytes"] = fwd["resident_bytes"] + rev["resident_bytes"]
        progress(f"scale {scale}: HITS graph in {out['create_s']:.1f} s")
        g.run(**kw)  # warm-up
        per_it = []
        for _ in range(runs):
            hubs, auth, st = g.run(**kw)
            assert st["iterations"] == iterations
            per_it.append(st["iterate_ms"] / iterations)
        out["hits_ms_per_iteration"] = float(np.median(per_it))
        out["hits_ms_per_iteration_all"] = per_it
        out["hits_edges_per_s"] = 2 * m / (out["hits_ms_per_iteration"] / 1e3)
        out["kernel_launches_per_iteration"] = st["kernel_launches"] / iterations
    progress(f"scale {scale}: HITS {out['hits_ms_per_iteration']:.3f} ms per iteration")
    with mg.PageRankGraph.from_arrays(n, f, t) as pg:
        pg.run(max_iterations=iterations, stop_epsilon=0.0)
        pr = []
        for _ in range(runs):
            _, st = pg.run(max_iterations=iterations, stop_epsilon=0.0)
            pr.append(st.iterate_ms / st.iterations)
    out["pagerank_ms_per_iteration"] = float(np.median(pr))
    out["pagerank_ms_per_iteration_all"] = pr
    out["ratio"] = out["hits_ms_per_iteration"] / out["pagerank_ms_per_iteration"]
    progress(f"scale {scale}: PageRank {out['pagerank_ms_per_iteration']:.3f} ms per iteration")
    oracle_need = 3 * 8 * n + 16 * m
    if scale > check_max_scale:
        out["max_rel_err"], out["check_skipped"] = None, f"scale > {check_max_scale}"
    elif available_host_bytes() < 1.2 * oracle_need:
        out["max_rel_err"] = None
        out["check_skipped"] = f"host memory: {available_host_bytes() / 2**30:.1f} GiB available"
    else:
        from test_hits_oracle import oracle_hits
        t0 = time.perf_counter()
        ref_h, ref_a, it, conv = oracle_hits(n, f, t, **kw)
        out["oracle_s"] = time.perf_counter() - t0
        out["max_rel_err"] = max(max_rel_err(hubs, ref_h), max_rel_err(auth, ref_a))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="22,24,26")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--iterations", type=int, default=20)
    ap.add_argument("--check-max-scale", type=int, default=24)
    args = ap.parse_args()
    result = {"workload": "hits", "card": card(), "gpu": []}
    for s in args.scales.split(","):
        result["gpu"].append(gpu_arm(int(s), args.runs, args.iterations, args.check_max_scale))
        print(json.dumps({"workload": result["workload"], "card": result["card"], "scale_result": result["gpu"][-1]}),
              flush=True)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Weighted shortest paths measurement: prints one JSON line per scale as soon as that scale is done (so an interrupted
run keeps what it finished), then one line with every scale together.

Per scale: an RMAT graph from the benchmark's generator (mg.rmat_edges_host, seed 42, 16 edges per vertex) built into
the BFS device graph, walked OUT and unbounded from vertex 0 with two seeded weight kinds (memgraph_b200.bfs.
splitmix_weights: "uniform" in [0, 1) with a 53-bit mantissa, "int" 1..16).  Per weight kind, one warm-up run, then the
median of --runs runs of mgb200_wsp_run.  Reported:
  ms                      median CUDA-event time (distance init .. last output written, no transfers)
  edges_per_s             m / t (input edges per second)
  relaxations_per_edge    (pass, vertex) lowerings / m
  buckets, rounds, delta  from the run's stats
  lower_bound_bytes       12 B per inspected entry (4 B id + 8 B weight) + 8 B per entry of offsets read twice per
                          vertex (2 x 8 B per reached vertex) + per-vertex distance traffic (8 B initialised, 8 B read
                          by the output pass, 8 + 4 B written out, 4 B hops initialised and read); NOT a bandwidth reached
  hbm_bound_fraction      (lower_bound_bytes / 3.35 TB/s, the H100 SXM data sheet) / t
  bfs_ms                  gpu_bfs (mgb200_bfs_run) on the same graph and source, median of --runs: a yardstick
  oracle_s / check        oracle/wsp_oracle.c (the cursor restatement) on the same input: its host time, and whether
                          total_weight is bit-identical and hops equal -- only at scales <= --check-max-scale and when
                          the host has the memory; check_skipped says why otherwise
A scale is skipped, with the reason, before anything is generated when its estimated peak does not fit: host memory
(HOST_BYTES_PER_EDGE) against MemAvailable, device memory (DEVICE_BYTES_PER_EDGE) against the card's total; a weight
sort that still does not fit on the device is reported skipped for that weight kind.  The card's name and power limit
are read in the same run.
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
# host peak per edge: the uint64 COO (16), the weights (8), splitmix_weights' uint64 temporaries (24) or
# set_weights' staging of weight bits and keys (16), whichever is larger, and the graph build's uint32 copy (8)
HOST_BYTES_PER_EDGE = 16 + 8 + 24 + 8
ORACLE_BYTES_PER_EDGE = 16 + 24  # its two edge lists, and a heap entry per pushed state (at most one per edge)
# device peak per edge: the graph build (sorted lists 8, keys 32, uint32 COO 8) or, later, the lists (8), the two weight
# arrays (16) and set_weights' staging (24) -- 48 either way, plus the sort's temporary
DEVICE_BYTES_PER_EDGE = 48 + 8


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
    return 12 * stats["entries_inspected"] + 16 * stats["reached"] + (8 + 8 + 8 + 4 + 4 + 4) * n


def progress(*what):
    print(*what, file=sys.stderr, flush=True)


def median_run(fn, runs, key):
    fn()  # warm-up: module load, allocations
    times, last = [], None
    for _ in range(runs):
        last = fn()
        times.append(last[-1][key])
    return float(np.median(times)), times, last


def device_total_bytes():
    import ctypes
    from memgraph_b200 import _native as N
    name, sms, total = ctypes.create_string_buffer(256), ctypes.c_int(0), ctypes.c_size_t(0)
    if N.lib().mgb200_device_info(0, name, 256, ctypes.byref(sms), ctypes.byref(total)):
        raise RuntimeError(N.lib().mgb200_last_error().decode())
    return total.value


def gpu_arm(scale, runs, check_max_scale):
    import memgraph_b200 as mg
    from memgraph_b200 import bfs
    from test_wsp_oracle import oracle_wsp, same_bits
    n, m = 1 << scale, 16 << scale
    need = HOST_BYTES_PER_EDGE * m + 64 * n
    device_need = DEVICE_BYTES_PER_EDGE * m + 128 * n
    out = {"scale": scale, "n": n, "m": m}
    if available_host_bytes() < 1.1 * need:
        out["skipped"] = (f"host memory: {available_host_bytes() / 2**30:.1f} GiB available, the COO, the weights and "
                          f"their staging need about {need / 2**30:.1f} GiB")
        return out
    if device_total_bytes() < 1.05 * device_need:
        out["skipped"] = (f"device memory: {device_total_bytes() / 2**30:.1f} GiB on the card, the graph, the weights "
                          f"and the weight sort need about {device_need / 2**30:.1f} GiB")
        return out
    t0 = time.perf_counter()
    f, t = mg.rmat_edges_host(scale, m, seed=42)
    g = bfs.BfsGraph(n, f, t)
    out["build_s"] = time.perf_counter() - t0
    progress(f"scale {scale}: graph built in {out['build_s']:.1f} s")
    with g:
        out["bfs_ms"], out["bfs_ms_all"], _ = median_run(lambda: g.distances(0, bfs.OUT), runs, "traverse_ms")
        out["weights"] = []
        for kind in ("uniform", "int"):
            w = bfs.splitmix_weights(m, kind)
            t0 = time.perf_counter()
            try:
                g.set_weights(f, t, w)
            except mg.MgB200Error as e:  # the weight sort's staging did not fit next to the resident graph
                out["weights"].append({"kind": kind, "skipped": str(e)})
                progress(f"scale {scale} {kind}: skipped: {e}")
                continue
            r = {"kind": kind, "set_weights_s": time.perf_counter() - t0}
            ms, all_ms, (dist, hops, stats) = median_run(lambda: g.weighted_distances(0, bfs.OUT), runs, "run_ms")
            t_s = ms / 1e3
            r.update({"ms": ms, "ms_all": all_ms, "edges_per_s": m / t_s, "relaxations_per_edge": stats["relaxations"] / m,
                      "buckets": stats["buckets"], "rounds": stats["rounds"], "delta": stats["delta"],
                      "lower_bound_bytes": lower_bound_bytes(n, stats),
                      "hbm_bound_fraction": lower_bound_bytes(n, stats) / HBM_BYTES_PER_S / t_s, "stats": stats})
            oracle_need = ORACLE_BYTES_PER_EDGE * m + 40 * n
            if scale > check_max_scale:
                r["check"], r["check_skipped"] = None, f"scale > {check_max_scale}"
            elif available_host_bytes() < 1.2 * oracle_need:
                r["check"] = None
                r["check_skipped"] = (f"host memory: {available_host_bytes() / 2**30:.1f} GiB available, the oracle needs "
                                      f"about {oracle_need / 2**30:.1f} GiB more")
            else:
                t0 = time.perf_counter()
                rc, odist, _, ohops, _ = oracle_wsp(n, f, t, w, 0, bfs.OUT, None)
                r["oracle_s"] = time.perf_counter() - t0
                r["check"] = bool(rc == 0 and same_bits(dist, odist) and np.array_equal(hops, ohops))
            progress(f"scale {scale} {kind}: {ms:.2f} ms, check {r['check']}")
            out["weights"].append(r)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="22,24,26")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--check-max-scale", type=int, default=24)
    args = ap.parse_args()
    result = {"workload": "weighted_shortest_paths", "card": card(), "gpu": []}
    for s in args.scales.split(","):
        result["gpu"].append(gpu_arm(int(s), args.runs, args.check_max_scale))
        print(json.dumps({"workload": result["workload"], "card": result["card"], "scale_result": result["gpu"][-1]}),
              flush=True)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Weakly connected components measurement: prints one JSON line.

GPU arm, per scale: a device-resident RMAT graph (the benchmark's generator, 16 edges per vertex), one warm-up run, then
the median of --runs runs of mgb200_wcc_run.  Reported per scale:
  build_s                 wall time of generating the edges and building the CSR + CSC on the device
  ms                      median CUDA-event time (parent init .. last label written)
  edges_per_s             m / t
  hbm_bound_fraction      (LOWER_BOUND_BYTES / 3.35 TB/s) / t, where LOWER_BOUND_BYTES = 4 * edges_inspected (each
                          inspected adjacency entry is a 4-byte id) + 4 * 8 * n (out- and in-offsets read in the
                          sampling and finish passes) + 4 * 4 * n (parent written by init, read by the label pass,
                          read and written by the final compression) + 8 * n (the labels written) -- a lower bound on
                          the HBM time as a share of the time taken; NOT a bandwidth reached
  stats                   the run's mgb200_wcc_stats
  check                   the output against oracle/wcc_oracle.c on the same edges in the same run (true / false), or
                          null with check_skipped saying why (not enough host memory for the uint64 COO and the oracle)
CPU arm: one CALL of the reference's own module (oracle/_ref, built by build() where a reference checkout exists)
against ours on the fake mgp host (tests/mgp_wcc_host.cpp), same RMAT input, wall time each, run in a child interpreter;
null where oracle/_ref was not built.  The card's name and power limit are read in the same run.
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
REF_WCC_MODULE_SO = os.path.join(REPO, "oracle", "_ref", "weakly_connected_components_reference.so")


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
    return 4 * stats["edges_inspected"] + 32 * n + 16 * n + 8 * n


def gpu_arm(scale, runs):
    import memgraph_b200 as mg
    from memgraph_b200 import _native as N
    from memgraph_b200.connectivity import BfsGraph, wcc_run
    from test_wcc_oracle import oracle_wcc
    lib = N.lib()
    n, m = 1 << scale, 16 << scale
    # uint64 COO (16 B/edge) + the oracle's undirected lists (8 B/edge) and offsets, queue, labels (28 B/vertex) + output
    check_bytes = 24 * m + 36 * n
    can_check = available_host_bytes() > 1.25 * check_bytes
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
    finally:
        lib.mgb200_device_free(0, d_from)
        lib.mgb200_device_free(0, d_to)
    out = {"scale": scale, "n": n, "m": m, "build_s": build_s}
    with g:
        wcc_run(g)  # warm-up: module load, allocations
        times, got, stats = [], None, None
        for _ in range(runs):
            got, stats = wcc_run(g)
            times.append(stats["run_ms"])
    t_s = float(np.median(times)) / 1e3
    out.update({"ms": float(np.median(times)), "ms_all": times, "edges_per_s": m / t_s,
                "lower_bound_bytes": lower_bound_bytes(n, stats),
                "hbm_bound_fraction": lower_bound_bytes(n, stats) / HBM_BYTES_PER_S / t_s, "stats": stats})
    if can_check:
        t0 = time.perf_counter()
        exp = oracle_wcc(n, f.astype(np.uint64), t.astype(np.uint64))
        out["check"] = bool(np.array_equal(got, exp))
        out["oracle_s"] = time.perf_counter() - t0
    else:
        out["check"] = None
        out["check_skipped"] = (f"host memory: {available_host_bytes() / 2**30:.1f} GiB available, the uint64 COO and "
                                f"the oracle need about {check_bytes / 2**30:.1f} GiB")
    return out


CPU_ARM_CODE = """
import json, sys, time
import numpy as np
sys.path[:0] = [%(tests)r, %(repo)r]
import memgraph_b200 as mg
import test_wcc_module as wm
scale = %(scale)d
n, m = 1 << scale, 16 << scale
f, t = mg.rmat_edges_host(scale, m, seed=42)
gids = np.arange(n, dtype=np.int64)
out = {"scale": scale, "n": n, "m": m}
with wm.Graph(gids, f.astype(np.int64), t.astype(np.int64)) as g:
    rows = {}
    for name, path in (("reference", wm.REF_WCC_MODULE_SO), ("gpu_module", wm.WCC_MODULE_SO)):
        with wm.Module(path) as module:
            module.call(g) if name == "gpu_module" else None  # the device module's first call also initialises CUDA
            t0 = time.perf_counter()
            rows[name] = wm.rows_of(*module.call(g))
            out[name + "_s"] = time.perf_counter() - t0
out["speedup"] = out["reference_s"] / out["gpu_module_s"]
out["rows_equal"] = bool(np.array_equal(rows["reference"], rows["gpu_module"]))
print(json.dumps(out))
"""


def cpu_arm(scale):
    if not os.path.exists(REF_WCC_MODULE_SO):
        return None
    code = CPU_ARM_CODE % {"tests": os.path.join(REPO, "tests"), "repo": REPO, "scale": scale}
    proc = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=3600)
    if proc.returncode:
        return {"error": (proc.stdout + proc.stderr)[-2000:]}
    return json.loads(proc.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="24,26")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--cpu-scale", type=int, default=20)
    args = ap.parse_args()
    result = {"workload": "weakly_connected_components", "card": card(),
              "gpu": [gpu_arm(int(s), args.runs) for s in args.scales.split(",")]}
    result["cpu"] = cpu_arm(args.cpu_scale)
    print(json.dumps(result))


if __name__ == "__main__":
    main()

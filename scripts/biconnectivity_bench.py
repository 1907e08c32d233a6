#!/usr/bin/env python3
"""Bridges and biconnected components measurement: prints one JSON line.

GPU arm, per scale: a device-resident RMAT graph (the benchmark's generator, 16 edges per vertex) built from the host
COO, one warm-up run, then the median of --runs runs of mgb200_biconnectivity_run.  Reported per scale:
  build_s                 wall time of generating the edges on the host and building the CSR + CSC on the device
  ms                      median CUDA-event time (first kernel .. last label written; the COO upload is not included)
  edges_per_s             m / t
  forest_depth            the BFS forest's deepest level: the forest and every sweep take one step per level
  lower_bound_bytes       4 * edges_inspected (each adjacency entry read is a 4-byte id, forest and low / high passes)
                          + 3 * 8 * m (the uint32 COO read by the root, link and classify passes) + 8 * m + m (the
                          labels and bridge flags written) + 16 * 8 * n (offsets read twice, ten 4-byte per-vertex
                          arrays written once and read once) -- a lower bound on the bytes moved
  hbm_bound_fraction      (lower_bound_bytes / 3.35 TB/s) / t -- the share of the time that traffic needs at the data
                          sheet's bandwidth; NOT a bandwidth reached
  stats                   the run's mgb200_biconnectivity_stats
  check                   the output against oracle/biconnectivity_oracle.c on the same edges (true / false), or null
                          with check_skipped saying why (not enough host memory)
A scale whose COO, outputs and oracle do not fit in host memory is reported skipped.
CPU arm: one CALL of each reference module (oracle/_ref, built by build() where a reference checkout exists) against
ours on the fake mgp host (tests/mgp_edge_host.cpp), same RMAT input at --cpu-scale, wall time each, in a child
interpreter.  The reference recurses once per DFS level, which overflows a default 8 MB stack on these graphs, so every
call runs in a thread with a 1 GiB stack (threading.stack_size).  Rows are compared as sets of bridges and as partitions
of the edges.  null where oracle/_ref was not built.  The card's name and power limit are read in the same run.
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
REF_SO = [os.path.join(REPO, "oracle", "_ref", f"{name}_reference.so") for name in ("bridges", "biconnected_components")]


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


def lower_bound_bytes(n, m, stats):
    return 4 * stats["edges_inspected"] + 24 * m + 9 * m + 128 * n


def gpu_arm(scale, runs):
    import memgraph_b200 as mg
    from memgraph_b200.connectivity import BfsGraph, biconnectivity_run
    from test_biconnectivity_oracle import oracle_biconnectivity
    n, m = 1 << scale, 16 << scale
    # uint64 COO (16 B/edge), the run's uint32 copy (8), outputs twice (18), the oracle's lists and stacks (40)
    need = 82 * m + 64 * n
    out = {"scale": scale, "n": n, "m": m}
    if available_host_bytes() < 1.1 * need:
        out["skipped"] = (f"host memory: {available_host_bytes() / 2**30:.1f} GiB available, the COO, outputs and "
                          f"oracle need about {need / 2**30:.1f} GiB")
        return out
    t0 = time.perf_counter()
    f, t = mg.rmat_edges_host(scale, m, seed=42)
    f, t = f.astype(np.uint64), t.astype(np.uint64)
    g = BfsGraph(n, f, t)
    out["build_s"] = time.perf_counter() - t0
    with g:
        biconnectivity_run(g, f, t)  # warm-up: module load, allocations
        times = []
        for _ in range(runs):
            bridge, bcc, stats = biconnectivity_run(g, f, t)
            times.append(stats["run_ms"])
    t_s = float(np.median(times)) / 1e3
    out.update({"ms": float(np.median(times)), "ms_all": times, "edges_per_s": m / t_s,
                "forest_depth": stats["forest_depth"], "lower_bound_bytes": lower_bound_bytes(n, m, stats),
                "hbm_bound_fraction": lower_bound_bytes(n, m, stats) / HBM_BYTES_PER_S / t_s, "stats": stats})
    t0 = time.perf_counter()
    exp_bridge, exp_bcc = oracle_biconnectivity(n, f, t)
    out["check"] = bool(np.array_equal(bridge, exp_bridge) and np.array_equal(bcc, exp_bcc))
    out["oracle_s"] = time.perf_counter() - t0
    return out


CPU_ARM_CODE = """
import json, sys, threading, time
import numpy as np
sys.path[:0] = [%(tests)r, %(repo)r]
import memgraph_b200 as mg
import test_biconnectivity_modules as bm
from test_biconnectivity_oracle import bcc_partition
scale = %(scale)d
n, m = 1 << scale, 16 << scale
f, t = mg.rmat_edges_host(scale, m, seed=42)
gids = np.arange(n, dtype=np.int64)
out = {"scale": scale, "n": n, "m": m, "stack_bytes": 1 << 30}


def call(path, g, key):
    with bm.Module(path) as module:
        if "reference" not in path:
            module.call(g)  # the device module's first call also initialises CUDA
        t0 = time.perf_counter()
        rows = module.call(g)
        out[key + "_s"] = time.perf_counter() - t0
    return rows


def run():
    with bm.Graph(gids, f.astype(np.int64), t.astype(np.int64)) as g:
        for name in ("bridges", "biconnected_components"):
            ref = call(bm.REF_MODULE_SO[name], g, name + "_reference")
            ours = call(bm.MODULE_SO[name], g, name + "_gpu_module")
            out[name + "_speedup"] = out[name + "_reference_s"] / out[name + "_gpu_module_s"]
            out[name + "_rows"] = [len(ref), len(ours)]
            same = bm.same_bridges(ref, ours) if name == "bridges" else bm.same_components(ref, ours)
            out[name + "_rows_equal"] = bool(same)


threading.stack_size(1 << 30)
th = threading.Thread(target=run)
th.start()
th.join()
print(json.dumps(out))
"""


def cpu_arm(scale):
    if not all(os.path.exists(p) for p in REF_SO):
        return None
    code = CPU_ARM_CODE % {"tests": os.path.join(REPO, "tests"), "repo": REPO, "scale": scale}
    proc = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=3600)
    if proc.returncode:
        return {"error": (proc.stdout + proc.stderr)[-2000:]}
    return json.loads(proc.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="22,24,26")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--cpu-scale", type=int, default=18)
    args = ap.parse_args()
    result = {"workload": "biconnectivity", "card": card(),
              "gpu": [gpu_arm(int(s), args.runs) for s in args.scales.split(",")]}
    result["cpu"] = cpu_arm(args.cpu_scale)
    print(json.dumps(result))


if __name__ == "__main__":
    main()

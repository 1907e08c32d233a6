#!/usr/bin/env python3
"""Builds kernel variants (different -D tunables) of libmgb200_pagerank.so for on-GPU sweeps.
Output: memgraph_b200/_build/variants/<name>/libmgb200_pagerank.so (select with MGB200_LIBRARY)."""
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from memgraph_b200 import build as B  # noqa: E402

VARIANTS = {
    "h_base": [], "h_pf8": ["-DMGB_HEAVY_PREFETCH=1"], "h_pf6": ["-DMGB_HEAVY_PREFETCH=1", "-DMGB_HEAVY_MIN_BLOCKS=6"],
    "h_pf5": ["-DMGB_HEAVY_PREFETCH=1", "-DMGB_HEAVY_MIN_BLOCKS=5"], "h_pf4": ["-DMGB_HEAVY_PREFETCH=1", "-DMGB_HEAVY_MIN_BLOCKS=4"],
    "h_b6": ["-DMGB_HEAVY_MIN_BLOCKS=6"], "h_b4": ["-DMGB_HEAVY_MIN_BLOCKS=4"],
    "h_u4pf8": ["-DMGB_HEAVY_PREFETCH=1", "-DMGB_UNROLL=4"], "h_u4b8": ["-DMGB_UNROLL=4"],
    # bound of a hot-only SELL walk (ranks wrong): every SELL gather from a label >= 2 M (the default block_from) reads
    # the zero slot instead, so the `sell_rows` class time is the walk without its HBM misses
    "sell_hot": ["-DMGB_SELL_HOT_ONLY_FROM=2097152"],
    # SELL walk registers (DESIGN.md §4): 4 CTAs per SM cap it at 64 registers and spill; 3 CTAs do not
    "s_b4": ["-DMGB_SELL_MIN_BLOCKS=4"], "s_b3": ["-DMGB_SELL_MIN_BLOCKS=3"], "s_u6": ["-DMGB_SELL_UNROLL=6", "-DMGB_SELL_MIN_BLOCKS=4"],
    "s_u4": ["-DMGB_SELL_UNROLL=4", "-DMGB_SELL_MIN_BLOCKS=4"],
    "s_u12b3": ["-DMGB_SELL_UNROLL=12", "-DMGB_SELL_MIN_BLOCKS=3"], "s_u16b2": ["-DMGB_SELL_UNROLL=16", "-DMGB_SELL_MIN_BLOCKS=2"],
    # SELL table kernel threads (one CTA per SM): 1024 caps it at 64 registers and spills, 768 does not; and the walk's
    # unroll at 768 threads (MGB_SELL_UNROLL also sets the plain kernel's)
    "t1024": ["-DMGB_TABLE_THREADS=1024"], "t768": ["-DMGB_TABLE_THREADS=768"],
    "t768_u6": ["-DMGB_TABLE_THREADS=768", "-DMGB_SELL_UNROLL=6"], "t768_u12": ["-DMGB_TABLE_THREADS=768", "-DMGB_SELL_UNROLL=12"],
    # the SELL walk's reads of staged values without L1 allocation (default: they may allocate)
    "stage_noalloc": ["-DMGB_STAGE_L1=0"],
}


def main():
    names = sys.argv[1:] or list(VARIANTS)
    objs = B.build_core()
    others = [o for o in objs if not o.endswith("pagerank_kernels.o")]
    for name in names:
        out = os.path.join(B.OUT, "variants", name)
        os.makedirs(out, exist_ok=True)
        obj = os.path.join(out, "pagerank_kernels.o")
        log = subprocess.run([B.NVCC] + B.NVCC_FLAGS + VARIANTS[name] + ["-c", os.path.join(B.CSRC, "pagerank_kernels.cu"), "-o", obj],
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if log.returncode:
            print(log.stdout)
            raise SystemExit(1)
        sell = ""
        lines = log.stdout.splitlines()
        for i, l in enumerate(lines):  # registers and spills of the SELL walks (plain, table) and the heavy-segment kernel
            if "Compiling entry function" in l and ("sell_rows_kernelILi0E" in l or "sell_rows_table_kernelILi0E" in l or
                                                    "heavy_segments_kernelILi0ELb0E" in l):
                sell += " | ".join(x.strip() for x in lines[i + 2:i + 4]) + "\n           "
        subprocess.run([B.NVCC, "-shared", "-cudart", "static", "-o", os.path.join(out, "libmgb200_pagerank.so"), obj] + others, check=True)
        print(f"{name:10s} {sell.rstrip()}")


if __name__ == "__main__":
    main()

"""Counting model of the heavy rows' tile class (graph_build.cu heavy_class and tile_slices, one partition): how many
in-edges of the heavy rows come from a source in the tiled prefix, how many (row, tile) chunks they make, and how long
the chunks are.

It relabels like the build (in-degree descending, out-degree descending, id ascending), so its counts equal the
`tiled_edges` / `tile_chunks` of PageRankGraph.info for the same edges and knobs (tests/test_gpu_tiles.py).

    python scripts/tile_model.py --scale 20 [--tile-labels 16384 --tile-hot-mb 16 --tile-chunk 256 --heavy-min 1024]
"""
import argparse
import json
import os
import sys

import numpy as np


def tile_model(n, frm, to, tile_labels=16384, tile_hot_mb=16, tile_chunk=256, heavy_min=1024):
    frm = np.asarray(frm, dtype=np.int64)
    to = np.asarray(to, dtype=np.int64)
    indeg = np.bincount(to, minlength=n)
    outdeg = np.bincount(frm, minlength=n)
    order = np.lexsort((np.arange(n), -outdeg, -indeg))  # sorted position -> vertex
    label = np.empty(n, dtype=np.int64)
    label[order] = np.arange(n)
    n_heavy = int(np.count_nonzero(indeg >= heavy_min))
    src, dst = label[frm], label[to]
    heavy = dst < n_heavy
    hot_labels = (tile_hot_mb << 20) // 8
    out = {"n": n, "m": len(frm), "heavy_rows": n_heavy, "heavy_edges": int(np.count_nonzero(heavy)),
           "tiled_edges": 0, "tile_chunks": 0, "tiles": 0, "chunk_length_histogram": {}}
    if tile_labels == 0:
        return out
    out["tiles"] = -(-min(hot_labels, n) // tile_labels)
    tiled = heavy & (src < hot_labels)
    pair = dst[tiled] * out["tiles"] + src[tiled] // tile_labels
    _, cnt = np.unique(pair, return_counts=True)
    chunks = -(-cnt // tile_chunk)
    full = cnt // tile_chunk
    lengths = np.concatenate([np.repeat(tile_chunk, int(full.sum())), (cnt % tile_chunk)[cnt % tile_chunk > 0]])
    edges = [1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024, 1 << 62]
    hist, _ = np.histogram(lengths, bins=edges)
    out["tiled_edges"] = int(tiled.sum())
    out["tile_chunks"] = int(chunks.sum())
    out["chunk_length_histogram"] = {f"[{lo},{hi})" if hi < 1 << 62 else f">={lo}": int(h)
                                     for lo, hi, h in zip(edges[:-1], edges[1:], hist)}
    out["edges_per_chunk"] = out["tiled_edges"] / max(out["tile_chunks"], 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=20)
    ap.add_argument("--edge-factor", type=int, default=16)
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--tile-labels", type=int, default=16384)
    ap.add_argument("--tile-hot-mb", type=int, default=16)
    ap.add_argument("--tile-chunk", type=int, default=256)
    ap.add_argument("--heavy-min", type=int, default=1024)
    args = ap.parse_args()
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import memgraph_b200 as mg
    n, m = 1 << args.scale, args.edge_factor << args.scale
    f, t = mg.rmat_edges_host(args.scale, m, seed=args.seed)
    print(json.dumps(tile_model(n, f, t, args.tile_labels, args.tile_hot_mb, args.tile_chunk, args.heavy_min)))


if __name__ == "__main__":
    main()

"""Counting model of the block class (graph_build.cu block_edges and block_slices, one partition): which in-edges of the
heavy rows come from a source label >= --block-from, how many (row, label block) chunks of at most --block-chunk edges
they make, in how many non-empty blocks, and how long the chunks are.  With --sell-blocks 1 (the default) it also counts
what putting the SELL rows into the class would move (measured slower and not built, DESIGN.md §4): their in-edges from
a source label >= --block-from that lies in a block the heavy rows launch, one chunk per (row, block) run, and the
SELL-32 padding of the layout with every column (`sell_pad_full`) and with the hot columns only (`sell_pad`). It also
counts the SELL entries the build stages (graph_build.cu sell_staging): the SELL rows' in-edges from a launched block,
in total (`stage_entries`) and per launched block in block order (`stage_entries_per_block`).

It relabels like the build (in-degree descending, out-degree descending, id ascending), so its counts equal the
`block_edges`, `block_chunks`, `blocks` and `stage_entries` of PageRankGraph.info for the same edges and knobs
(tests/test_gpu_block_gather.py, tests/test_gpu_sell_stage.py).

    python scripts/block_model.py --scale 22 [--block-from 2097152 --block-labels 2097152 --block-chunk 16 --heavy-min 1024]
"""
import argparse
import json
import os
import sys

import numpy as np


def block_model(n, frm, to, block_from=2 << 20, block_labels=2 << 20, block_chunk=16, heavy_min=1024, max_blocks=4096,
                sell_blocks=1):
    frm = np.asarray(frm, dtype=np.int64)
    to = np.asarray(to, dtype=np.int64)
    indeg = np.bincount(to, minlength=n)
    outdeg = np.bincount(frm, minlength=n)
    order = np.lexsort((np.arange(n), -outdeg, -indeg))  # sorted position -> vertex
    label = np.empty(n, dtype=np.int64)
    label[order] = np.arange(n)
    n_heavy = int(np.count_nonzero(indeg >= heavy_min))
    src, dst = label[frm], label[to]
    out = {"n": n, "m": len(frm), "heavy_rows": n_heavy, "heavy_edges": int(np.count_nonzero(dst < n_heavy)),
           "block_edges": 0, "block_chunks": 0, "blocks": 0, "chunk_length_histogram": {},
           "stage_entries": 0, "stage_entries_per_block": []}
    sell = sell_counts(n, indeg, src, dst, n_heavy, heavy_min, None, block_from, 1) if sell_blocks else None
    if block_labels == 0 or n <= block_from:
        if sell:
            out.update(sell)
        return out
    labels = max(block_labels, -(-(n - block_from) // max_blocks))  # the build keeps <= max_blocks blocks
    cold = (dst < n_heavy) & (src >= block_from)
    nb = -(-(n - block_from) // labels)
    pair, cnt = np.unique(dst[cold] * nb + (src[cold] - block_from) // labels, return_counts=True)
    lengths = np.concatenate([np.repeat(block_chunk, int((cnt // block_chunk).sum())), (cnt % block_chunk)[cnt % block_chunk > 0]])
    edges = [1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1 << 62]
    hist, _ = np.histogram(lengths, bins=edges)
    out["block_edges"] = int(cold.sum())
    out["block_chunks"] = int((-(-cnt // block_chunk)).sum())
    out["blocks"] = int(len(np.unique(pair % nb)))
    out["chunk_length_histogram"] = {f"[{lo},{hi})" if hi < 1 << 62 else f">={lo}": int(h)
                                     for lo, hi, h in zip(edges[:-1], edges[1:], hist)}
    out["edges_per_chunk"] = out["block_edges"] / max(out["block_chunks"], 1)
    out.update(stage_counts(indeg, src, dst, n_heavy, heavy_min, np.unique(pair % nb), block_from, labels))
    if sell_blocks:
        out.update(sell_counts(n, indeg, src, dst, n_heavy, heavy_min, np.unique(pair % nb), block_from, labels))
    return out


def stage_counts(indeg, src, dst, n_heavy, heavy_min, launched, block_from, labels):
    """SELL entries staged by the passes of the launched blocks (`launched`: block numbers, ascending)."""
    sell_rows = int(np.count_nonzero((indeg >= 1) & (indeg < heavy_min)))
    in_sell = (dst >= n_heavy) & (dst < n_heavy + sell_rows)
    blk = np.where(src >= block_from, (src - block_from) // labels, -1)
    staged = in_sell & np.isin(blk, launched)
    per_block = [int(np.count_nonzero(staged & (blk == b))) for b in launched]
    return {"stage_entries": int(staged.sum()), "stage_entries_per_block": per_block}


def sell_counts(n, indeg, src, dst, n_heavy, heavy_min, launched, block_from, labels):
    """SELL rows' block chunks: edges from a launched block (`launched`: block numbers, None = no block class)."""
    sell_rows = int(np.count_nonzero((indeg >= 1) & (indeg < heavy_min)))
    in_sell = (dst >= n_heavy) & (dst < n_heavy + sell_rows)
    deg = np.bincount(dst[in_sell] - n_heavy, minlength=sell_rows)  # descending: rows are sorted by in-degree
    cold = np.zeros(len(src), dtype=bool)
    if launched is not None and len(launched):
        blk = np.where(src >= block_from, (src - block_from) // labels, -1)
        cold = in_sell & np.isin(blk, launched)
    rows, blocks = dst[cold] - n_heavy, (src[cold] - block_from) // labels
    pair = np.unique(rows * (len(launched) and int(launched.max()) + 1) + blocks) if cold.any() else np.zeros(0, np.int64)
    hot = deg - np.bincount(rows, minlength=sell_rows)
    slices = -(-sell_rows // 32)
    pad = np.zeros(slices * 32, dtype=np.int64)

    def padding(d):
        pad[:] = 0
        pad[:sell_rows] = d
        return int((pad.reshape(slices, 32).max(axis=1) * 32).sum() - d.sum())
    bn = int(launched.max()) + 1 if launched is not None and len(launched) else 1
    per_block = np.bincount(pair % bn, minlength=bn) if len(pair) else np.zeros(bn, np.int64)
    return {"sell_rows": sell_rows, "sell_block_edges": int(cold.sum()), "sell_block_chunks": int(len(pair)),
            "sell_block_rows_max": int(per_block.max()) if len(pair) else 0,
            "sell_pad_full": padding(deg), "sell_pad": padding(hot)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=20)
    ap.add_argument("--edge-factor", type=int, default=16)
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--block-from", type=int, default=2 << 20)
    ap.add_argument("--block-labels", type=int, default=2 << 20)
    ap.add_argument("--block-chunk", type=int, default=16)
    ap.add_argument("--heavy-min", type=int, default=1024)
    ap.add_argument("--sell-blocks", type=int, default=1)
    args = ap.parse_args()
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import memgraph_b200 as mg
    n, m = 1 << args.scale, args.edge_factor << args.scale
    f, t = mg.rmat_edges_host(args.scale, m, seed=args.seed)
    print(json.dumps(block_model(n, f, t, args.block_from, args.block_labels, args.block_chunk, args.heavy_min,
                                 sell_blocks=args.sell_blocks)))


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Regenerates ``scc_cases.json`` in this directory with networkx; the tests use the committed file, so they pin the
partition to networkx's on machines without it.

The reference's ``nxalg.strongly_connected_components`` (query_modules/nxalg.py) builds a networkx ``MultiDiGraph`` of
every vertex and every edge of the graph and returns ``networkx.strongly_connected_components`` of it.  Each graph of
tests/test_scc_oracle.py (``handmade_graphs`` and ``seeded_graphs``) is built the same way here, and networkx's
components are stored canonically: component[v] = the rank of the smallest vertex of v's component among all
components' smallest vertices.
"""
import json
import os
import sys

import networkx as nx
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def networkx_components(n, f, t):
    g = nx.MultiDiGraph()
    g.add_nodes_from(range(n))
    g.add_edges_from(zip([int(x) for x in f], [int(x) for x in t]))
    smallest = np.empty(n, dtype=np.int64)
    for comp in nx.strongly_connected_components(g):
        smallest[list(comp)] = min(comp)
    rank = {v: i for i, v in enumerate(sorted(set(smallest.tolist())))}
    return [rank[int(s)] for s in smallest]


def main():
    sys.path[:0] = [os.path.dirname(HERE)]
    from test_scc_oracle import handmade_graphs, seeded_graphs
    handmade = []
    for name, n, edges in handmade_graphs():
        handmade.append({"name": name, "n": n, "edges": [list(e) for e in edges],
                         "components": networkx_components(n, [a for a, _ in edges], [b for _, b in edges])})
    seeded = [{"name": name, "n": n, "m": len(f), "components": networkx_components(n, f, t)}
              for name, n, f, t in seeded_graphs()]
    out = {"source": f"networkx {nx.__version__} strongly_connected_components on a MultiDiGraph of all vertices",
           "handmade": handmade, "seeded": seeded}
    with open(os.path.join(HERE, "scc_cases.json"), "w") as fh:
        json.dump(out, fh, separators=(",", ":"))
        fh.write("\n")
    print("wrote scc_cases.json")


if __name__ == "__main__":
    main()

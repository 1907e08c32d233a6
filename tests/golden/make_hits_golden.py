#!/usr/bin/env python3
"""Extracts the reference's cuGraph HITS e2e fixtures (mage/tests/e2e/hits_test/test_cugraph_*: input.cyp + test.yml)
into tests/golden/hits_e2e.json.  Usage: make_hits_golden.py <memgraph checkout>.

Two input styles occur: `MERGE (a:Node {id: x}) MERGE (b:Node {id: y}) MERGE (a)-[:R]->(b)` (the relationship is
de-duplicated) and `CREATE (a1:Node {id: 1, name: 'A1'})` followed by `MATCH (a:Node {id: x}), (b:Node {id: y})
CREATE (a)-[:R]->(b)` (every line is an edge).  Vertices are listed in order of first appearance."""
import json
import os
import re
import sys

import yaml

REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("MG_REFERENCE", "")
BASE = os.path.join(REF, "mage", "tests", "e2e", "hits_test")
HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_ARGS = [100, 1e-5, True]  # the module's registered defaults


def parse_graph(cyp):
    nodes, edges, merged = [], [], set()
    for line in cyp.splitlines():
        line = line.strip()
        if not line or line.startswith("//"):
            continue
        ids = [int(x) for x in re.findall(r"\{id: (\d+)", line)]
        if "->" not in line:
            for v in ids:  # CREATE (a1:Node {id: 1, name: 'A1'})
                if v not in nodes:
                    nodes.append(v)
            continue
        a, b = ids
        for v in (a, b):
            if v not in nodes:
                nodes.append(v)
        if re.search(r"MERGE \(\w+\)-", line):  # MERGE de-duplicates the relationship, CREATE does not
            if (a, b) in merged:
                continue
            merged.add((a, b))
        edges.append([a, b])
    return nodes, edges


def parse_args(query):
    m = re.search(r"cugraph\.hits\.get\(([^)]*)\)", query)
    args = list(DEFAULT_ARGS)
    if m and m.group(1).strip():
        for i, tok in enumerate(t.strip() for t in m.group(1).split(",")):
            args[i] = int(tok) if i == 0 else float(tok) if i == 1 else tok.upper() == "TRUE"
    return args


def main():
    out = []
    for name in sorted(os.listdir(BASE)):
        if not name.startswith("test_cugraph"):
            continue
        d = os.path.join(BASE, name)
        cyp_path = os.path.join(d, "input.cyp")
        cyp = open(cyp_path).read() if os.path.exists(cyp_path) else ""
        spec = yaml.safe_load(open(os.path.join(d, "test.yml")))
        nodes, edges = parse_graph(cyp)
        expected = [[row["node_id"], float(row["hubs"]), float(row["authorities"])] for row in (spec.get("output") or [])]
        out.append({"name": name[len("test_cugraph_"):], "nodes": nodes, "edges": edges,
                    "args": parse_args(spec["query"]), "expected": expected,
                    "source": f"mage/tests/e2e/hits_test/{name}"})
    json.dump(out, open(os.path.join(HERE, "hits_e2e.json"), "w"), indent=1)
    print(len(out), "fixtures")


if __name__ == "__main__":
    main()

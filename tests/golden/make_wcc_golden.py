#!/usr/bin/env python3
"""Regenerates the weakly connected components fixtures in this directory from a memgraph checkout (MG_REFERENCE) and
oracle/_ref as built by oracle/wcc.mk; the tests use the committed files.

* ``wcc_e2e_cases.json``       <- mage/tests/e2e/weakly_connected_components_test/* (5 cases).  Each case is a list of
  query steps, one graph per step: the two online cases run three queries, after adding the second component, after
  adding the isolated vertex 6 and after deleting it.  Nodes are listed in creation order (= the view's visit order).
* ``wcc_ref_module_rows.json`` <- the reference's own module (oracle/_ref/weakly_connected_components_reference.so)
  through tests/mgp_wcc_host.cpp on the graphs of tests/test_wcc_module.py:wcc_scattered_graphs: its signature and
  sha256 of its (gid, component) rows sorted by gid.
"""
import json
import os
import re
import subprocess
import sys

import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("MG_REFERENCE", "")
E2E_DIR = "mage/tests/e2e/weakly_connected_components_test"

EDGE = re.compile(r"MERGE \(a:Node \{id: (\d+)\}\) MERGE \(b:Node \{id: (\d+)\}\) CREATE \(a\)-\[:RELATION\]->\(b\)")
NODE = re.compile(r"MERGE \(a:Node \{id: (\d+)\}\)")
DELETE = re.compile(r"MATCH \(a:Node \{id: (\d+)\}\) DELETE a")


def apply(statements, nodes, edges):
    """Runs the fixture's Cypher statements on (nodes in creation order, edges by node id)."""
    for stmt in (s.strip() for s in statements.split(";")):
        if not stmt:
            continue
        if m := EDGE.fullmatch(stmt):
            a, b = int(m.group(1)), int(m.group(2))
            for v in (a, b):
                if v not in nodes:
                    nodes.append(v)
            edges.append([a, b])
        elif m := NODE.fullmatch(stmt):
            if int(m.group(1)) not in nodes:
                nodes.append(int(m.group(1)))
        elif m := DELETE.fullmatch(stmt):
            v = int(m.group(1))
            assert all(v not in e for e in edges), "DELETE of a vertex with edges"
            nodes.remove(v)
        else:
            raise ValueError(stmt)


def wcc_online_case(name):
    d = os.path.join(REF, E2E_DIR, name)
    queries = yaml.safe_load(open(os.path.join(d, "input.cyp")))
    expected = yaml.safe_load(open(os.path.join(d, "test.yml")))
    nodes, edges, steps = [], [], []
    apply(queries.get("setup", ""), nodes, edges)
    assert len(queries["queries"]) == len(expected)
    for q, exp in zip(queries["queries"], expected):
        apply(q, nodes, edges)
        steps.append({"nodes": list(nodes), "edges": [list(e) for e in edges], "output": exp["output"]})
    return {"name": name, "steps": steps}


def wcc_cases():
    out = []
    for name in sorted(os.listdir(os.path.join(REF, E2E_DIR))):
        d = os.path.join(REF, E2E_DIR, name)
        spec = yaml.safe_load(open(os.path.join(d, "test.yml")))
        if isinstance(spec, list):
            out.append(wcc_online_case(name))
            continue
        nodes, edges = [], []
        apply(open(os.path.join(d, "input.cyp")).read(), nodes, edges)
        out.append({"name": name, "steps": [{"nodes": nodes, "edges": edges, "output": spec["output"]}]})
    assert len(out) == 5, [c["name"] for c in out]
    return {"source": E2E_DIR + "/*", "cases": out}


def wcc_ref_module_rows():
    """In a child interpreter: the host library must be the only one loaded (tests/_bc_host.py)."""
    code = """
import json
import test_wcc_module as wm
out = {"source": "oracle/_ref/weakly_connected_components_reference.so through libmgp_wcc_host.so", "graphs": []}
with wm.Module(wm.REF_WCC_MODULE_SO) as module:
    out["signature"] = module.signature()
    for name, gids, src, dst in wm.wcc_scattered_graphs():
        with wm.Graph(gids, src, dst) as g:
            rows = wm.rows_of(*module.call(g))
        out["graphs"].append({"name": name, "rows": len(rows), "components": int(rows[:, 1].max()) + 1,
                              "rows_sha256": wm.rows_sha256(rows)})
print(json.dumps(out))
"""
    tests = os.path.dirname(HERE)
    proc = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True,
                          env=dict(os.environ, PYTHONPATH=os.pathsep.join([tests, os.path.dirname(tests)])))
    return json.loads(proc.stdout)


def main():
    if not os.path.isdir(REF):
        sys.exit("reference checkout not present; golden fixtures are committed, nothing to do")
    for name, fn in [("wcc_e2e_cases.json", wcc_cases), ("wcc_ref_module_rows.json", wcc_ref_module_rows)]:
        with open(os.path.join(HERE, name), "w") as f:
            json.dump(fn(), f, separators=(",", ":"))
            f.write("\n")
        print("wrote", name)


if __name__ == "__main__":
    main()

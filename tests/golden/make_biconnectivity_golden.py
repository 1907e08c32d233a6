#!/usr/bin/env python3
"""Regenerates the bridges / biconnected components fixtures in this directory from a memgraph checkout (MG_REFERENCE)
and oracle/_ref as built by oracle/biconnectivity.mk; the tests use the committed files.

* ``biconnectivity_e2e_cases.json``      <- mage/tests/e2e/bridges_test/* (3 cases) and
  mage/tests/e2e/biconnected_components_test/* (1 case).  Nodes are listed in creation order (= the view's visit order).
* ``biconnectivity_unit_graphs.json``    <- the handmade graphs of mage/cpp/bridges_module/bridges_test.cpp and
  mage/cpp/biconnected_components_module/biconnected_components_test.cpp with their expected answers, as data (the
  generated ones -- cycles, random trees, random graphs -- are left out).
* ``biconnectivity_ref_module_rows.json`` <- the reference's own modules (oracle/_ref/{bridges,biconnected_components}_
  reference.so) through tests/mgp_edge_host.cpp on the graphs of
  tests/test_biconnectivity_modules.py:scattered_graphs: their signatures and raw rows (bcc_id or 0, from gid, to gid).
"""
import ast
import json
import os
import re
import subprocess
import sys

import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("MG_REFERENCE", "")
E2E = {"bridges": "mage/tests/e2e/bridges_test", "biconnected_components": "mage/tests/e2e/biconnected_components_test"}
UNIT = {"bridges": "mage/cpp/bridges_module/bridges_test.cpp",
        "biconnected_components": "mage/cpp/biconnected_components_module/biconnected_components_test.cpp"}

EDGE = re.compile(r"MERGE \(a:Node \{id: (\d+)\}\) MERGE \(b:Node \{id: (\d+)\}\) CREATE \(a\)-\[:RELATION\]->\(b\)")


def e2e_cases():
    out = []
    for module, rel in E2E.items():
        for name in sorted(os.listdir(os.path.join(REF, rel))):
            d = os.path.join(REF, rel, name)
            nodes, edges = [], []
            for stmt in (s.strip() for s in open(os.path.join(d, "input.cyp")).read().split(";")):
                if not stmt or stmt == "MATCH (n) DETACH DELETE n":
                    continue
                m = EDGE.fullmatch(stmt)
                if not m:
                    raise ValueError(stmt)
                a, b = int(m.group(1)), int(m.group(2))
                nodes += [v for v in (a, b) if v not in nodes]
                edges.append([a, b])
            spec = yaml.safe_load(open(os.path.join(d, "test.yml")))
            out.append({"module": module, "name": name, "nodes": nodes, "edges": edges, "output": spec["output"]})
    assert len(out) == 4, [c["name"] for c in out]
    return {"source": " and ".join(v + "/*" for v in E2E.values()), "cases": out}


def braced(text):
    """A C++ braced initializer of integers -> nested Python lists."""
    return ast.literal_eval(text.replace("{", "[").replace("}", "]"))


def balanced(text, start):
    """The braced group that opens at text[start]."""
    depth = 0
    for i in range(start, len(text)):
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        if depth == 0:
            return text[start:i + 1]
    raise ValueError("unbalanced")


def unit_graphs():
    out = {}
    for module, rel in UNIT.items():
        src = open(os.path.join(REF, rel)).read()
        cases = []
        for m in re.finditer(r"TEST\((\w+), (\w+)\) \{(.*?)\n\}", src, re.S):
            body = m.group(3)
            g = re.search(r"BuildGraph\(\s*(\d+),\s*\{", body)
            if not g:
                continue  # generated graphs
            edges = braced(balanced(body, g.end() - 1))
            case = {"name": m.group(2), "n": int(g.group(1)), "edges": edges}
            if module == "bridges":
                c = re.search(r"CheckBridges\(\s*bridges,\s*\{", body)
                if c:
                    case["bridges"] = braced(balanced(body, c.end() - 1))
                    case["bridge_count"] = len(case["bridges"])
                else:
                    case["bridge_count"] = int(re.search(r"ASSERT_EQ\((\d+), bridges\.size\(\)\)", body).group(1))
                    case["bridge_edge_ids"] = [int(x) for x in re.findall(r"ASSERT_EQ\(bridges\[\d+\]\.id, (\d+)\)", body)]
            else:
                c = re.search(r"CheckBCC\(\s*BCC,\s*\{", body)
                case["components"] = braced(balanced(body, c.end() - 1))
            cases.append(case)
        out[module] = cases
    out["source"] = " and ".join(UNIT.values())
    return out


def ref_module_rows():
    """In a child interpreter: the host library must be the only one loaded (tests/_bc_host.py)."""
    code = """
import json
import test_biconnectivity_modules as bm
out = {"source": "oracle/_ref/{bridges,biconnected_components}_reference.so through libmgp_edge_host.so", "modules": {}}
for name, path in bm.REF_MODULE_SO.items():
    with bm.Module(path) as module:
        entry = {"signature": module.signature(), "graphs": []}
        for gname, gids, src, dst in bm.scattered_graphs():
            with bm.Graph(gids, src, dst) as g:
                entry["graphs"].append({"name": gname, "rows": module.call(g).tolist()})
    out["modules"][name] = entry
print(json.dumps(out))
"""
    tests = os.path.dirname(HERE)
    proc = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True,
                          env=dict(os.environ, PYTHONPATH=os.pathsep.join([tests, os.path.dirname(tests)])))
    return json.loads(proc.stdout)


def main():
    if not os.path.isdir(REF):
        sys.exit("reference checkout not present; golden fixtures are committed, nothing to do")
    for name, fn in [("biconnectivity_e2e_cases.json", e2e_cases), ("biconnectivity_unit_graphs.json", unit_graphs),
                     ("biconnectivity_ref_module_rows.json", ref_module_rows)]:
        with open(os.path.join(HERE, name), "w") as f:
            json.dump(fn(), f, separators=(",", ":"))
            f.write("\n")
        print("wrote", name)


if __name__ == "__main__":
    main()

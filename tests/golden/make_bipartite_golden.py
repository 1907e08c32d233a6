#!/usr/bin/env python3
"""Regenerates ``bipartite_cases.json`` in this directory from a memgraph checkout (MG_REFERENCE) and oracle/_ref as
built by oracle/bipartite.mk; the tests use the committed file.

* ``e2e``    <- mage/tests/e2e/bipartite_matching_test/* (4 cases).  Nodes are listed in creation order.
* ``unit``   <- the fixed graphs of mage/cpp/bipartite_matching_module/bipartite_matching_test.cpp, as data (the random
  complete bipartite graphs and the timing case are left out).  Handmade* call MaximumMatching on two 1-based vertex
  sets A and B; they are stored as graphs with A's vertex i at i - 1 and B's vertex j at |A| + j - 1.  The four colouring
  checks state only bipartite or not; their expected count is the reference module's.
* ``seeded`` <- the reference module's answer on every graph of tests/test_bipartite_oracle.py:seeded_graphs.

The reference module is called through tests/mgp_wcc_host.cpp in a child interpreter (tests/_bc_host.py), on a thread
with a 1 GiB stack: its recursive DFS overflows the default 8 MB one from a few thousand vertices on.
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
E2E = "mage/tests/e2e/bipartite_matching_test"
UNIT = "mage/cpp/bipartite_matching_module/bipartite_matching_test.cpp"
EDGE = re.compile(r"MERGE \(a:Node \{id: (\d+)\}\) MERGE \(b:Node \{id: (\d+)\}\) CREATE \(a\)-\[:RELATION\]->\(b\)")


def braced(text):
    """A C++ braced initializer of integers -> nested Python lists."""
    return ast.literal_eval(text.replace("{", "[").replace("}", "]"))


def e2e_cases():
    out = []
    for name in sorted(os.listdir(os.path.join(REF, E2E))):
        d = os.path.join(REF, E2E, name)
        nodes, edges = [], []
        cyp = os.path.join(d, "input.cyp")
        for stmt in (s.strip() for s in (open(cyp).read() if os.path.exists(cyp) else "").split(";")):
            if not stmt:
                continue
            m = EDGE.fullmatch(stmt)
            if not m:
                raise ValueError(stmt)
            a, b = int(m.group(1)), int(m.group(2))
            nodes += [v for v in (a, b) if v not in nodes]
            edges.append([a, b])
        spec = yaml.safe_load(open(os.path.join(d, "test.yml")))
        [row] = spec["output"]
        out.append({"name": name, "nodes": nodes, "edges": edges, "expected": row["maximum_bipartite_matching"]})
    assert len(out) == 4, [c["name"] for c in out]
    return out


def unit_cases():
    src = open(os.path.join(REF, UNIT)).read()
    out = []
    for m in re.finditer(r"TEST\((\w+), (\w+)\) \{(.*?)\n\}", src, re.S):
        name, body = m.group(2), m.group(3)
        expected = re.search(r"ASSERT_EQ\(max_match, (\d+)\)", body)
        g = re.search(r"BuildGraph\(\s*(\d+),\s*(\{.*?\})\);", body, re.S)
        sets = re.search(r"bipartite_edges = (\{.*?\});", body, re.S)
        if g:
            case = {"name": name, "n": int(g.group(1)), "edges": braced(g.group(2))}
        elif sets and expected:
            pairs = braced(sets.group(1))
            a = max(p[0] for p in pairs)
            case = {"name": name, "n": a + max(p[1] for p in pairs),
                    "edges": [[i - 1, a + j - 1] for i, j in pairs]}
        else:
            continue  # generated graphs
        case["expected"] = int(expected.group(1)) if expected else None
        out.append(case)
    assert len(out) == 16, [c["name"] for c in out]
    return out


def reference_answers(graphs):
    """[(n, from, to)] -> the reference module's answers, computed in a child interpreter on a 1 GiB-stack thread."""
    code = """
import json, sys, threading
import test_bipartite_module as bm
graphs = json.load(sys.stdin)
out = []
def run():
    with bm.Module(bm.REF_MODULE_SO) as ref:
        for n, f, t in graphs:
            out.append(bm.call(ref, n, f, t))
threading.stack_size(1 << 30)
th = threading.Thread(target=run)
th.start()
th.join()
print(json.dumps(out))
"""
    tests = os.path.dirname(HERE)
    proc = subprocess.run([sys.executable, "-c", code], input=json.dumps(graphs), capture_output=True, text=True,
                          check=True, env=dict(os.environ, PYTHONPATH=os.pathsep.join([tests, os.path.dirname(tests)])))
    return json.loads(proc.stdout)


def main():
    if not os.path.isdir(REF):
        sys.exit("reference checkout not present; golden fixtures are committed, nothing to do")
    sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
    from test_bipartite_oracle import seeded_graphs
    e2e, unit = e2e_cases(), unit_cases()
    answers = reference_answers([[c["n"], [e[0] for e in c["edges"]], [e[1] for e in c["edges"]]] for c in unit])
    for case, got in zip(unit, answers):
        assert case["expected"] in (None, got), (case["name"], case["expected"], got)
        case["expected"] = got
    seeded = seeded_graphs()
    answers = reference_answers([[n, [int(x) for x in f], [int(x) for x in t]] for _, n, f, t in seeded])
    out = {"source": f"{E2E}/*, {UNIT} and oracle/_ref/bipartite_matching_reference.so through libmgp_wcc_host.so",
           "e2e": e2e, "unit": unit,
           "seeded": [{"name": name, "n": n, "m": len(f), "expected": got}
                      for (name, n, f, t), got in zip(seeded, answers)]}
    with open(os.path.join(HERE, "bipartite_cases.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))
        f.write("\n")
    print("wrote bipartite_cases.json")


if __name__ == "__main__":
    main()

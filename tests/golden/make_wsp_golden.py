"""Records tests/golden/wsp_unit_cases.json: the reference's own expectations for the weighted shortest path expansion
(ExpandWeightedShortestPathCursor, src/query/plan/operator.cpp:2917-3267), transcribed from its tests as data.  The
engine operator cannot be compiled on its own, so these fixtures are what pins oracle/wsp_oracle.c to the reference.

Sources:
  QueryPlanExpandWeightedShortestPath (tests/unit/query_plan_match_filter_return.cpp:1872-2223): five vertices v0..v4
    (dense ids = creation order), edges 0->1 (5), 1->4 (5), 0->2 (3), 2->3 (3), 3->4 (3), 4->0 (12), all DOUBLE; the
    expansion starts at v0.  Basic, EdgeDirection OUT / IN, UpperBound none / 1 / 2 / 3 (3: plus v5 and 4->5 with the
    INTEGER weight 2), NonNumericWeight (4->5 'not a number'), NegativeWeight (4->5 -10), NegativeUpperBound (-1).
  tests/gql_behave/tests/memgraph_V1/features/memgraph_wshortest.feature, the scenarios whose weight is one edge
    property and which have no filter: "upper bound", "resulting edge list", "weight not a number", "negative weight".
    Vertices in CREATE order; the error scenarios match every start vertex, so the case starts at the one whose
    expansion raises (vertex 0).

Each case: n, edges [from, to, weight, type] (type "double" / "int" / "string"), start, direction (0 OUT, 1 IN,
2 BOTH), upper_bound (null = none), and either rows [vertex, total_weight, size(le) or null when the test does not
check it] in the reference's yield order, or error {kind, message}.  Run: python tests/golden/make_wsp_golden.py
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
UNIT = "tests/unit/query_plan_match_filter_return.cpp"
FEATURE = "tests/gql_behave/tests/memgraph_V1/features/memgraph_wshortest.feature"

BASE = [[0, 1, 5.0, "double"], [1, 4, 5.0, "double"], [0, 2, 3.0, "double"], [2, 3, 3.0, "double"],
        [3, 4, 3.0, "double"], [4, 0, 12.0, "double"]]
DEPTH_MESSAGE = "Maximum depth in weighted shortest path expansion must be at least 1."


def unit(name, line, direction, upper_bound, rows=None, extra=None, error=None):
    edges = BASE + ([extra] if extra else [])
    case = {"name": name, "origin": f"{UNIT}:{line}", "n": 6 if extra else 5, "edges": edges, "start": 0,
            "direction": direction, "upper_bound": upper_bound}
    case.update({"rows": rows} if error is None else {"error": error})
    return case


def behave(name, line, edges, upper_bound, rows=None, error=None):
    case = {"name": name, "origin": f"{FEATURE}:{line}", "n": 4, "edges": edges, "start": 0, "direction": 0,
            "upper_bound": upper_bound}
    case.update({"rows": rows} if error is None else {"error": error})
    return case


def cases():
    out = [
        unit("Basic", 2033, 2, 1000, [[2, 3, 1], [1, 5, 1], [3, 6, 2], [4, 9, 3]]),
        unit("EdgeDirection OUT", 2065, 0, 1000, [[2, 3, None], [1, 5, None], [3, 6, None], [4, 9, None]]),
        unit("EdgeDirection IN", 2065, 1, 1000, [[4, 12, None], [3, 15, None], [1, 17, None], [2, 18, None]]),
        unit("UpperBound none", 2141, 2, None, [[2, 3, None], [1, 5, None], [3, 6, None], [4, 9, None]]),
        unit("UpperBound 2", 2141, 2, 2, [[2, 3, None], [1, 5, None], [3, 6, None], [4, 10, None]]),
        unit("UpperBound 1", 2141, 2, 1, [[2, 3, None], [1, 5, None], [4, 12, None]]),
        unit("UpperBound 3", 2141, 2, 3, [[2, 3, None], [1, 5, None], [3, 6, None], [4, 9, None], [5, 12, None]],
             extra=[4, 5, 2, "int"]),
        unit("NonNumericWeight", 2200, 2, 1000, extra=[4, 5, "not a number", "string"],
             error={"kind": "non_numeric", "message": "Weight must be numeric or a Duration, got string."}),
        unit("NegativeWeight", 2210, 2, 1000, extra=[4, 5, -10, "int"],
             error={"kind": "negative", "message": "Weight must be non-negative, got -10."}),
        unit("NegativeUpperBound", 2221, 2, -1, error={"kind": "upper_bound", "message": DEPTH_MESSAGE}),
        behave("upper bound", 3, [[0, 1, 1, "int"], [1, 2, 1, "int"], [0, 3, 1, "int"]], 1,
               [[1, 1, None], [3, 1, None]]),
        behave("resulting edge list", 32, [[0, 1, 1, "int"], [1, 2, 2, "int"], [0, 3, 4, "int"]], 10,
               [[1, 1, 1], [2, 3, 2], [3, 4, 1]]),
        behave("weight not a number", 93, [[0, 1, "not a number", "string"], [1, 2, 2, "int"], [0, 3, 3, "int"]], 10,
               error={"kind": "non_numeric", "message": "Weight must be numeric or a Duration, got string."}),
        behave("negative weight", 106, [[0, 1, -1, "int"], [1, 2, 2, "int"], [0, 3, 3, "int"]], 10,
               error={"kind": "negative", "message": "Weight must be non-negative, got -1."}),
    ]
    return out


if __name__ == "__main__":
    with open(os.path.join(HERE, "wsp_unit_cases.json"), "w") as f:
        json.dump({"cases": cases()}, f, indent=1)
        f.write("\n")

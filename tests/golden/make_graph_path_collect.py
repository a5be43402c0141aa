"""Writes graph_path_collect.json, the fixture of the per-row `+collect` language tests, from a SurrealDB source checkout:

  python tests/golden/make_graph_path_collect.py <surrealdb checkout>

Output (committed):
  graph_path_collect.json
    cases   {file: {"statements": [...], "results": [...]}} of language-tests/tests/language/graph/path_collect.surql,
            over the records of language-tests/tests/datasets/graph.surql (graph_relations.json, graph_filters.json)
"""
import json
import os
import re
import sys

from make_graph_filters import HERE, statements

FILES = ["path_collect.surql"]


def main(ref):
    lt = os.path.join(ref, "language-tests", "tests")
    cases = {}
    for f in FILES:
        txt = open(os.path.join(lt, "language", "graph", f)).read()
        head, body = txt.split("*/", 1)
        cases[f] = {"statements": statements(body), "results": re.findall(r'^value = "(.*)"$', head, flags=re.M)}
        assert len(cases[f]["statements"]) == len(cases[f]["results"]), f
    json.dump({"cases": cases}, open(os.path.join(HERE, "graph_path_collect.json"), "w"), indent=1)
    print(sum(len(c["statements"]) for c in cases.values()), "statements")


if __name__ == "__main__":
    main(sys.argv[1])

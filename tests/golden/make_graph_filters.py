"""Writes graph_filters.json, the fixture of the WHERE-filtered graph hops, from a SurrealDB source checkout:

  python tests/golden/make_graph_filters.py <surrealdb checkout>

Output (committed):
  graph_filters.json
    edge_props   {edge record id: fields} of every `RELATE a->tb:id->b SET ...` in
                 language-tests/tests/datasets/graph.surql
    node_props   {record id: fields} of every `CREATE tb:id SET ...` there
    cases        {file: {"statements": [...], "results": [...]}} of language-tests/tests/language/graph/
                 filter_edge_properties.surql, filter_target_nodes.surql and filter_combined.surql
  Field values: numbers and strings as JSON, d"..." as {"datetime": "..."}, record ids as {"record": "tb:id"},
  NONE as null, arrays as lists.
"""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
FILES = ["filter_edge_properties.surql", "filter_target_nodes.surql", "filter_combined.surql"]


def split_top(s, sep=","):
    """split at `sep` outside quotes and brackets"""
    out, depth, quote, cur = [], 0, None, ""
    for ch in s:
        if quote:
            quote = None if ch == quote else quote
        elif ch in "\"'":
            quote = ch
        elif ch in "[{(":
            depth += 1
        elif ch in "]})":
            depth -= 1
        elif ch == sep and depth == 0:
            out.append(cur)
            cur = ""
            continue
        cur += ch
    if cur.strip():
        out.append(cur)
    return [x.strip() for x in out]


def value(v):
    v = v.strip()
    if v == "NONE":
        return None
    if v.startswith("d\""):
        return {"datetime": v[2:-1]}
    if v[0] in "\"'":
        return v[1:-1]
    if v.startswith("["):
        return [value(x) for x in split_top(v[1:-1])]
    if re.fullmatch(r"-?\d+", v):
        return int(v)
    if re.fullmatch(r"-?\d+\.\d*", v):
        return float(v)
    if re.fullmatch(r"\w+:\w+", v):
        return {"record": v}
    raise ValueError(f"unhandled value {v!r}")


def fields(set_clause):
    out = {}
    for a in split_top(set_clause):
        k, v = a.split("=", 1)
        out[k.strip()] = value(v)
    return out


def statements(body):
    lines = [l for l in body.splitlines() if l.strip() and not l.strip().startswith("--")]
    return [" ".join(s.split()) + ";" for s in " ".join(lines).split(";") if s.strip()]


def main(ref):
    lt = os.path.join(ref, "language-tests", "tests")
    ds = open(os.path.join(lt, "datasets", "graph.surql")).read()
    ds = "\n".join(l for l in ds.split("*/", 1)[1].splitlines() if not l.strip().startswith("--"))
    edge_props, node_props = {}, {}
    for m in re.finditer(r"RELATE\s+\w+:\w+->(\w+:\w+)->\w+:\w+(?:\s+SET\s+([^;]*))?;", ds):
        edge_props[m.group(1)] = fields(m.group(2)) if m.group(2) else {}
    for m in re.finditer(r"CREATE\s+(\w+:\w+)\s+SET\s+([^;]*);", ds, flags=re.S):
        node_props[m.group(1)] = fields(" ".join(m.group(2).split()))
    cases = {}
    for f in FILES:
        txt = open(os.path.join(lt, "language", "graph", f)).read()
        head, body = txt.split("*/", 1)
        cases[f] = {"statements": statements(body), "results": re.findall(r'^value = "(.*)"$', head, flags=re.M)}
        assert len(cases[f]["statements"]) == len(cases[f]["results"]), f
    json.dump({"edge_props": edge_props, "node_props": node_props, "cases": cases},
              open(os.path.join(HERE, "graph_filters.json"), "w"), indent=1)
    print(len(edge_props), "edge records,", len(node_props), "records,",
          sum(len(c["statements"]) for c in cases.values()), "statements")


if __name__ == "__main__":
    main(sys.argv[1])

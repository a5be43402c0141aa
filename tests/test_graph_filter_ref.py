"""The CPU restatement of the WHERE-filtered graph hop (tests/graph_filter_ref.py) against the unfiltered oracle and the
reference's language tests filter_edge_properties.surql, filter_target_nodes.surql and filter_combined.surql (over
datasets/graph.surql; extracted into tests/golden/graph_filters.json by tests/golden/make_graph_filters.py)."""
import json
import os
import re

import numpy as np
import pytest

import graph_filter_ref as R
from oracle import pyoracle as O
from surrealdb_b200.graph import GraphStore, pack_bits

HERE = os.path.dirname(os.path.abspath(__file__))
REL = json.load(open(os.path.join(HERE, "golden", "graph_relations.json")))["relations"]
F = json.load(open(os.path.join(HERE, "golden", "graph_filters.json")))

# every WHERE condition of the three files, translated by hand; a field the record lacks (NONE) compares false
COND = {
    "hours > 20": lambda p: p.get("hours", -1) > 20,
    "hours >= 25": lambda p: p.get("hours", -1) >= 25,
    "hours > 15": lambda p: p.get("hours", -1) > 15,
    'strength = "strong"': lambda p: p.get("strength") == "strong",
    'level = "expert"': lambda p: p.get("level") == "expert",
    'since > d"2021-01-01"': lambda p: "since" in p and p["since"]["datetime"] > "2021-01-01",
    'role = "lead" AND hours >= 25': lambda p: p.get("role") == "lead" and p.get("hours", -1) >= 25,
    'role = "contributor"': lambda p: p.get("role") == "contributor",
    'role = "lead"': lambda p: p.get("role") == "lead",
    'status = "active"': lambda p: p.get("status") == "active",
    "priority = 1": lambda p: p.get("priority") == 1,
    "priority > 1": lambda p: p.get("priority", -1) > 1,
    'status = "active" AND priority <= 2': lambda p: p.get("status") == "active" and "priority" in p and p["priority"] <= 2,
    'category = "backend"': lambda p: p.get("category") == "backend",
    'category = "database"': lambda p: p.get("category") == "database",
    'category = "frontend"': lambda p: p.get("category") == "frontend",
}


def target_pred(table, cond):
    """`(table WHERE cond)` as the target of a hop: a record of that table satisfying cond"""
    return lambda p: p["id"].startswith(table + ":") and COND[cond](p)


def parse_hops(rest):
    """`->(e WHERE c)->(n WHERE c)->e->n...` -> [(direction, edge_table, edge_pred, target_pred), ...]"""
    segs = re.findall(r"->(?:\((\w+) WHERE ([^)]*)\)|(\w+))", rest)
    assert "".join("->" + (f"({a} WHERE {b})" if a else c) for a, b, c in segs) == rest, rest
    hops = []
    for (ea, ec, eb), (ta, tc, _tb) in zip(segs[0::2], segs[1::2]):
        hops.append(("out", ea or eb, COND[ec] if ea else None, target_pred(ta, tc) if ta else None))
    return hops


def fmt(names):
    return "[" + ", ".join(names) + "]"


def statements():
    """every statement of the three files as (statement, expected result, evaluate(lookup) -> result string), where
    lookup(start, hops) runs the filtered chain and returns record ids"""
    out = []
    for f, case in F["cases"].items():
        for stmt, want in zip(case["statements"], case["results"]):
            m = re.fullmatch(r"(\w+:\w+)(->.*);", stmt)
            if m:
                start, hops = m.group(1), parse_hops(m.group(2))
                out.append((stmt, want, lambda lookup, s=start, h=hops: fmt(lookup([s], h))))
                continue
            # SELECT id, name, ->(e WHERE c)->node.name AS alias FROM a, b;  (fields print in key order)
            m = re.fullmatch(r"SELECT id, name, (->.*?)\.name AS (\w+) FROM ([\w:, ]+);", stmt)
            assert m, stmt
            hops, alias, starts = parse_hops(m.group(1)), m.group(2), [s.strip() for s in m.group(3).split(",")]

            def select(lookup, hops=hops, alias=alias, starts=starts):
                rows = []
                for s in starts:
                    row = {"id": s, "name": f"'{F['node_props'][s]['name']}'",
                           alias: "[" + ", ".join(f"'{F['node_props'][t]['name']}'" for t in lookup([s], hops)) + "]"}
                    rows.append("{ " + ", ".join(f"{k}: {row[k]}" for k in sorted(row)) + " }")
                return "[" + ", ".join(rows) + "]"
            out.append((stmt, want, select))
    return out


def store(ctx=None):
    return GraphStore(ctx, [(r["src"], r["edge_tb"], r["edge_id"], r["dst"]) for r in REL],
                      edge_props=F["edge_props"], node_props=F["node_props"])


def test_reference_restatement_reproduces_the_filter_language_tests():
    st = store()

    def lookup(start, hops):
        chain = []
        for d, tb, ep, tp in hops:
            rp, ci = st.csr_arrays(tb, d)
            em, tm = st.hop_masks(tb, d, ep, tp)
            chain.append((rp, ci, None if em is None else pack_bits(em), None if tm is None else pack_bits(tm)))
        return st.to_names(R.chain(chain, st.ids(start)))
    cases = statements()
    for stmt, want, run in cases:
        assert run(lookup) == want, stmt
    assert len(cases) == 19  # 7 edge-property, 6 target-node and 6 combined statements: every one of the three files


def test_edge_record_map_follows_the_csr_order():
    st = store()
    for tb, d in (("works_on", "out"), ("works_on", "in"), ("knows", "both"), (None, "out"), (("knows", "works_on"), "in")):
        rp, ci = st.csr_arrays(tb, d)
        recs = st.edge_records(tb, d)
        assert len(recs) == ci.size
        by_id = {f"{r['edge_tb']}:{r['edge_id']}": r for r in REL}
        for v in range(rp.size - 1):
            for p in range(int(rp[v]), int(rp[v + 1])):
                r = by_id[recs[p]]
                ends = {st.idx[r["src"]], st.idx[r["dst"]]}
                assert v in ends and int(ci[p]) in ends, (tb, d, v, p)
    # `<->`: each edge record at two positions of each endpoint's row, so an edge mask marks both
    recs = st.edge_records("knows", "both")
    assert all(recs.count(e) == 4 for e in set(recs))


def rand_csr(rng, n, m, hub=0):
    src = np.concatenate([rng.integers(0, n, m), np.zeros(hub, np.int64)])
    dst = rng.integers(0, n, src.size)
    order = np.argsort(src, kind="stable")
    rp = np.zeros(n + 1, np.uint64)
    rp[1:] = np.cumsum(np.bincount(src, minlength=n))
    return rp, dst[order].astype(np.uint32)


def pruned(rp, ci, em, tm):
    """the CSR with the failing positions removed"""
    keep = em & tm[ci]
    rows = np.repeat(np.arange(rp.size - 1), np.diff(rp.astype(np.int64)))
    rp2 = np.zeros(rp.size, np.uint64)
    rp2[1:] = np.cumsum(np.bincount(rows[keep], minlength=rp.size - 1))
    return rp2, ci[keep]


@pytest.mark.parametrize("limit", [0, 1, 3])
@pytest.mark.parametrize("density", [0.0, 0.01, 0.5, 1.0])
def test_filtered_hop_is_the_unfiltered_hop_minus_failing_positions(limit, density):
    rng = np.random.default_rng(int(density * 100) + limit)
    n = 500
    rp, ci = rand_csr(rng, n, 6000, hub=3000)
    frontier = rng.integers(0, n, 400).astype(np.uint32)
    frontier[:3] = 0  # the hub, three times
    em = rng.random(ci.size) < density
    tm = rng.random(n) < max(density, 0.3)
    eb, tb = pack_bits(em), pack_bits(tm)
    assert np.array_equal(R.bits_of(eb, ci.size), em) and np.array_equal(R.bits_of(tb, n), tm)
    got = R.hop(rp, ci, frontier, eb, tb, limit)
    assert np.array_equal(got, O.graph_hop(*pruned(rp, ci, em, tm), frontier, limit))
    if limit == 0:  # positions of the unfiltered output, in order: the filtered output is exactly the passing ones
        pos = np.concatenate([np.arange(int(rp[v]), int(rp[v + 1])) for v in frontier])
        assert np.array_equal(got, O.graph_hop(rp, ci, frontier)[em[pos] & tm[ci[pos]]])
    ones = np.ones(ci.size, bool)
    assert np.array_equal(R.hop(rp, ci, frontier, pack_bits(ones), None, limit), O.graph_hop(rp, ci, frontier, limit))
    assert np.array_equal(R.hop(rp, ci, frontier, None, None, limit), O.graph_hop(rp, ci, frontier, limit))
    # edge-only and target-only conditions
    assert np.array_equal(R.hop(rp, ci, frontier, eb, None, limit),
                          O.graph_hop(*pruned(rp, ci, em, np.ones(n, bool)), frontier, limit))
    assert np.array_equal(R.hop(rp, ci, frontier, None, tb, limit), O.graph_hop(*pruned(rp, ci, ones, tm), frontier, limit))


@pytest.mark.parametrize("inclusive", [False, True])
def test_filtered_collect_is_collect_over_the_pruned_csr(inclusive):
    rng = np.random.default_rng(7 + inclusive)
    n = 2000
    rp, ci = rand_csr(rng, n, 16000)
    em, tm = rng.random(ci.size) < 0.6, rng.random(n) < 0.7
    total = 0
    for start, mn, mx in ((5, 1, 0), (77, 2, 4), (123, 1, 3), (9, 3, 0)):
        want = O.graph_collect(*pruned(rp, ci, em, tm), [start], mn, mx, inclusive)
        got = R.collect(rp, ci, [start], pack_bits(em), pack_bits(tm), mn, mx, inclusive)
        assert np.array_equal(got, want), (start, mn, mx)
        total += got.size
    assert total > 1000


def test_pack_bits():
    m = np.zeros(70, bool)
    m[[0, 31, 32, 69]] = True
    w = pack_bits(m)
    assert w.dtype == np.uint32 and w.tolist() == [0x80000001, 1, 1 << 5]
    assert pack_bits(w) is not None and pack_bits(w).tolist() == w.tolist()
    assert pack_bits(np.zeros(0, bool)).size == 0
    with pytest.raises(TypeError):
        pack_bits(np.zeros(3, np.int32))

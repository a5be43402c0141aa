"""Host-side mirror of the graph-scan operators on top of the C ABI.

  CsrGraph            sdb_graph: device CSR of one (direction, edge table)
  GraphStore          what the Rust shim builds from the `~` edge-pointer keys (key/graph/mod.rs:122-137):
                      per (direction, edge table) a CSR whose rows list, per source record, the targets in KV
                      key order of the connecting edge records (SURVEY appendix A8)
  GraphStore.lookup   LookupPart over a fused GraphEdgeScan chain (exec/parts/lookup.rs:139-170,
                      exec/planner/idiom.rs:161-193): multiset, order-preserving
  GraphStore.collect  `.{min..max+collect[+inclusive]}` (exec/operators/recursion/collect.rs:74-143)
  GraphStore.recurse  default `.{min..max}` recursion (exec/operators/recursion/default.rs:75-133)
  GraphStore.lookup_filtered / collect_filtered / recurse_filtered
                      the same with WHERE conditions on the edge and target records, evaluated into bitmaps
                      (hop_masks) for sdb_graph_expand_filtered / sdb_graph_collect_filtered
  GraphStore.lookup_batch / collect_batch
                      LookupPart::evaluate_batch (exec/parts/lookup.rs:96-112): lookup / collect of every row of a
                      ValueBatch, optionally filtered, in one sdb_graph_expand_batch / sdb_graph_collect_batch call
  GraphEdgeScan       the operator itself: new(input, direction, edge_tables, output_mode, version).with_limit(n)
                      (exec/operators/scan/graph.rs:89-147) -- name(), attrs(), execute()
"""
import ctypes as C

import numpy as np

from . import _lib as L


class CsrGraph:
    def __init__(self, ctx, row_ptr, col_idx):
        self.ctx = ctx
        rp = np.ascontiguousarray(row_ptr, np.uint64)
        ci = np.ascontiguousarray(col_idx, np.uint32)
        self.n_rows = rp.size - 1
        self.h = C.c_void_p()
        L.check(L.lib().sdb_graph_load_csr(ctx.h, self.n_rows, C.c_void_p(rp.ctypes.data),
                                           C.c_void_p(ci.ctypes.data) if ci.size else None, C.byref(self.h)))

    def close(self):
        if self.h:
            L.lib().sdb_graph_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CsrGraphShard(CsrGraph):
    """rows [row_lo, row_hi) of an n_rows_total-row CSR on this context's GPU (sdb_graph_load_csr_shard).  `row_ptr` /
    `col_idx` are the WHOLE graph's arrays (host): the slice is cut and rebased here.  expand / expand_device / collect
    on shard handles are collective over the context's communicator -- one thread or process per rank."""

    def __init__(self, ctx, row_ptr, col_idx, row_lo, row_hi):
        self.ctx = ctx
        rp_all = np.asarray(row_ptr, np.uint64)
        self.n_rows = rp_all.size - 1
        e0, e1 = int(rp_all[row_lo]), int(rp_all[row_hi])
        rp = np.ascontiguousarray(rp_all[row_lo:row_hi + 1] - np.uint64(e0))
        ci = np.ascontiguousarray(np.asarray(col_idx, np.uint32)[e0:e1])
        self.row_lo, self.row_hi = int(row_lo), int(row_hi)
        self.h = C.c_void_p()
        L.check(L.lib().sdb_graph_load_csr_shard(ctx.h, self.n_rows, self.row_lo, self.row_hi, C.c_void_p(rp.ctypes.data),
                                                 C.c_void_p(ci.ctypes.data) if ci.size else None, C.byref(self.h)))


def _take(out, n):
    if not out or n.value == 0:
        return np.zeros(0, np.uint32)
    arr = np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_uint32)), shape=(n.value,)).copy()
    L.lib().sdb_free(out)
    return arr


def expand(hops, frontier, per_source_limit=0):
    """sdb_graph_expand: apply the CSR hops in order to the frontier (multiset semantics)."""
    fr = np.ascontiguousarray(frontier, np.uint32)
    arr = (C.c_void_p * len(hops))(*[g.h for g in hops])
    out, n = C.c_void_p(), C.c_uint64()
    L.check(L.lib().sdb_graph_expand(arr, len(hops), C.c_void_p(fr.ctypes.data) if fr.size else None, fr.size,
                                     int(per_source_limit), C.byref(out), C.byref(n)))
    return _take(out, n)


def expand_device(ctx, hops, d_frontier, n_frontier, per_source_limit=0):
    """sdb_graph_expand_device: frontier and result stay in HBM. -> (device pointer (int), count); free with
    device_free(ctx, ptr)."""
    arr = (C.c_void_p * len(hops))(*[g.h for g in hops])
    out, n = C.c_void_p(), C.c_uint64()
    L.check(L.lib().sdb_graph_expand_device(arr, len(hops), C.c_void_p(d_frontier), int(n_frontier), int(per_source_limit),
                                            C.byref(out), C.byref(n)))
    return (out.value or 0), n.value


def device_free(ctx, ptr):
    if ptr:
        L.lib().sdb_device_free(ctx.h, C.c_void_p(ptr))


def collect(graph, start, min_depth=1, max_depth=0, inclusive=False):
    st = np.ascontiguousarray(start, np.uint32)
    out, n = C.c_void_p(), C.c_uint64()
    L.check(L.lib().sdb_graph_collect(graph.h, C.c_void_p(st.ctypes.data) if st.size else None, st.size, int(min_depth),
                                      int(max_depth), int(bool(inclusive)), C.byref(out), C.byref(n)))
    return _take(out, n)


class HopFilter(C.Structure):
    """sdb_hop_filter"""
    _fields_ = [("edge_bits", C.c_void_p), ("target_bits", C.c_void_p)]


def pack_bits(mask):
    """a bitmap for the filtered calls: uint32 words (bit i = bit i % 32 of word i // 32) are taken as they are, a bool
    array (one entry per CSR position or node id) is packed"""
    a = np.asarray(mask)
    if a.dtype == np.uint32:
        return np.ascontiguousarray(a)
    if a.dtype != np.bool_:
        raise TypeError(f"bitmap: expected uint32 words or a bool mask, got {a.dtype}")
    b = np.packbits(a, bitorder="little")
    b = np.concatenate([b, np.zeros(-b.size % 4, np.uint8)])
    return b.view("<u4").astype(np.uint32)


def _filters(filters, n, on_device):
    """(edge_bits, target_bits) or None per hop -> (sdb_hop_filter array, the packed host arrays it points into)"""
    if len(filters) != n:
        raise ValueError(f"{len(filters)} filters for {n} hops")
    arr, keep = (HopFilter * n)(), []
    for h, f in enumerate(filters):
        for name, m in zip(("edge_bits", "target_bits"), f or (None, None)):
            if m is None:
                continue
            if on_device:  # a device pointer (int) or a tensor
                setattr(arr[h], name, int(m.data_ptr()) if hasattr(m, "data_ptr") else int(m))
            else:
                w = pack_bits(m)
                keep.append(w)
                setattr(arr[h], name, w.ctypes.data if w.size else None)
    return arr, keep


def expand_filtered(hops, filters, frontier, per_source_limit=0):
    """sdb_graph_expand_filtered: expand() with a WHERE condition per hop.  filters: per hop None or (edge_bits,
    target_bits), each None, a bool mask (per CSR position / per node id) or packed uint32 words."""
    fr = np.ascontiguousarray(frontier, np.uint32)
    arr = (C.c_void_p * len(hops))(*[g.h for g in hops])
    farr, _keep = _filters(filters, len(hops), False)
    out, n = C.c_void_p(), C.c_uint64()
    L.check(L.lib().sdb_graph_expand_filtered(arr, farr, len(hops), C.c_void_p(fr.ctypes.data) if fr.size else None, fr.size,
                                              int(per_source_limit), C.byref(out), C.byref(n)))
    return _take(out, n)


def expand_filtered_device(ctx, hops, filters, d_frontier, n_frontier, per_source_limit=0):
    """sdb_graph_expand_filtered_device: filters hold DEVICE bitmaps (pointers or tensors of packed uint32 words).
    -> (device pointer (int), count); free with device_free(ctx, ptr)."""
    arr = (C.c_void_p * len(hops))(*[g.h for g in hops])
    farr, _keep = _filters(filters, len(hops), True)
    out, n = C.c_void_p(), C.c_uint64()
    L.check(L.lib().sdb_graph_expand_filtered_device(arr, farr, len(hops), C.c_void_p(d_frontier), int(n_frontier),
                                                     int(per_source_limit), C.byref(out), C.byref(n)))
    return (out.value or 0), n.value


def collect_filtered(graph, filt, start, min_depth=1, max_depth=0, inclusive=False):
    """sdb_graph_collect_filtered: collect() whose every level is the filtered hop; filt = (edge_bits, target_bits)"""
    st = np.ascontiguousarray(start, np.uint32)
    farr, _keep = _filters([filt], 1, False)
    out, n = C.c_void_p(), C.c_uint64()
    L.check(L.lib().sdb_graph_collect_filtered(graph.h, farr, C.c_void_p(st.ctypes.data) if st.size else None, st.size,
                                               int(min_depth), int(max_depth), int(bool(inclusive)), C.byref(out), C.byref(n)))
    return _take(out, n)


def _docs(docs):
    """a batch of documents: a list of per-document id arrays, or (ids, doc_off) -> (ids uint32, doc_off uint64)"""
    if isinstance(docs, tuple):
        ids, off = docs
        return np.ascontiguousarray(ids, np.uint32), np.ascontiguousarray(off, np.uint64)
    parts = [np.asarray(d, np.uint32).ravel() for d in docs]
    off = np.zeros(len(parts) + 1, np.uint64)
    off[1:] = np.cumsum([p.size for p in parts], dtype=np.uint64)
    ids = np.concatenate(parts) if parts else np.zeros(0, np.uint32)
    return np.ascontiguousarray(ids, np.uint32), off


def _split(ids, off):
    return [ids[int(off[d]):int(off[d + 1])] for d in range(off.size - 1)]


def _ptr(a):
    return C.c_void_p(a.ctypes.data) if a.size else None


def expand_batch(hops, docs, per_source_limit=0, filters=None):
    """sdb_graph_expand_batch: expand() of every document of the batch in one call.  docs: a list of per-document id
    arrays or (ids, doc_off); filters: None or, per hop, as in expand_filtered.  -> one array per document"""
    ids, off = _docs(docs)
    arr = (C.c_void_p * len(hops))(*[g.h for g in hops])
    farr, _keep = _filters(filters, len(hops), False) if filters is not None else (None, None)
    out, n = C.c_void_p(), C.c_uint64()
    out_off = np.zeros(off.size, np.uint64)
    L.check(L.lib().sdb_graph_expand_batch(arr, farr, len(hops), _ptr(ids), ids.size, C.c_void_p(off.ctypes.data),
                                           off.size - 1, int(per_source_limit), C.byref(out),
                                           C.c_void_p(out_off.ctypes.data), C.byref(n)))
    return _split(_take(out, n), out_off)


def expand_batch_device(ctx, hops, d_frontier, n_frontier, d_doc_off, n_docs, d_out_doc_off, per_source_limit=0,
                        filters=None):
    """sdb_graph_expand_batch_device: frontier, doc_off (n_docs + 1 uint64), the bitmaps and the result in HBM; the
    result's boundaries are written to d_out_doc_off (n_docs + 1 uint64).  -> (device pointer (int), count); free with
    device_free(ctx, ptr)."""
    arr = (C.c_void_p * len(hops))(*[g.h for g in hops])
    farr, _keep = _filters(filters, len(hops), True) if filters is not None else (None, None)
    out, n = C.c_void_p(), C.c_uint64()
    L.check(L.lib().sdb_graph_expand_batch_device(arr, farr, len(hops), C.c_void_p(d_frontier), int(n_frontier),
                                                  C.c_void_p(d_doc_off), int(n_docs), int(per_source_limit), C.byref(out),
                                                  C.c_void_p(d_out_doc_off), C.byref(n)))
    return (out.value or 0), n.value


def collect_batch(graph, docs, min_depth=1, max_depth=0, inclusive=False, filt=None):
    """sdb_graph_collect_batch: collect() of every document's start ids, each with its own first-seen set, in one
    call; filt: None or (edge_bits, target_bits) as in collect_filtered.  -> one array per document"""
    ids, off = _docs(docs)
    farr, _keep = _filters([filt], 1, False) if filt is not None else (None, None)
    out, n = C.c_void_p(), C.c_uint64()
    out_off = np.zeros(off.size, np.uint64)
    L.check(L.lib().sdb_graph_collect_batch(graph.h, farr, _ptr(ids), ids.size, C.c_void_p(off.ctypes.data), off.size - 1,
                                            int(min_depth), int(max_depth), int(bool(inclusive)), C.byref(out),
                                            C.c_void_p(out_off.ctypes.data), C.byref(n)))
    return _split(_take(out, n), out_off)


def last_collect_table(graph):
    """diagnostics of the last collect_batch on this graph: {peak_bytes, grows, repeated_passes, splits}"""
    b, g, r, s = C.c_uint64(), C.c_uint32(), C.c_uint32(), C.c_uint32()
    L.lib().sdb_graph_last_collect_table(graph.h, C.byref(b), C.byref(g), C.byref(r), C.byref(s))
    return {"peak_bytes": b.value, "grows": g.value, "repeated_passes": r.value, "splits": s.value}


def _key_order(rid_key):
    """storekey order of a RecordIdKey (val/record_id.rs:181-192): numbers (numeric) before strings (bytes)"""
    if isinstance(rid_key, (int, np.integer)):
        return (0, int(rid_key), b"")
    return (1, 0, str(rid_key).encode())


class GraphStore:
    """CSR snapshots of a set of RELATE edges: relations = iterable of (src, edge_table, edge_id, dst) with
    record ids like 'person:alice'.  For WHERE-filtered hops, edge_props maps an edge record id ('works_on:alice_db')
    and node_props a node record id to its fields (a dict); records without an entry have no fields."""

    def __init__(self, ctx, relations, edge_props=None, node_props=None):
        self.ctx = ctx
        rel = list(relations)
        self.names = sorted({r[0] for r in rel} | {r[3] for r in rel})
        self.idx = {n: i for i, n in enumerate(self.names)}
        self._rel = rel
        self._csr = {}
        self.edge_props = dict(edge_props or {})
        self.node_props = dict(node_props or {})

    def csr_arrays(self, edge_table, direction):
        return self._csr_build(edge_table, direction)[:2]

    def edge_records(self, edge_table, direction):
        """the edge record id behind every CSR position of csr_arrays(edge_table, direction), from the same sort (a
        `<->` CSR lists each edge record at two positions of each endpoint's row)"""
        rel = self._csr_build(edge_table, direction)[2]
        return [f"{self._rel[r][1]}:{self._rel[r][2]}" for r in rel]

    def _csr_build(self, edge_table, direction):
        """(row_ptr, col_idx) of one `node <dir> edge_table <dir> node` step, neighbours in the order the reference's
        KV scan yields them: per source the graph keys sort by (direction, edge table, edge record key)
        (key/graph/mod.rs:122-137).  edge_table=None is the `?` wildcard (all edge tables, scan/graph.rs:303-311); a tuple of
        names = one key range per table, scanned in the listed order (scan/graph.rs:312-324).  direction: 'out' (->), 'in' (<-) or 'both' (<->): GraphEdgeScan scans In, then
        Out (exec/operators/scan/graph.rs:203-207), and the second `<->` of the pair yields both endpoints of every
        edge record, In pointer (the edge's source node) first."""
        adj = [[] for _ in self.names]
        for ri, (src, tb, eid, dst) in enumerate(self._rel):
            if edge_table is None:  # the `?` wildcard: one range over every edge table, i.e. key order by table name
                tkey = tb.encode()
            elif isinstance(edge_table, (tuple, list)):  # one range per listed table, scanned in the listed order
                if tb not in edge_table:
                    continue
                tkey = list(edge_table).index(tb)
            else:
                if tb != edge_table:
                    continue
                tkey = 0
            ek = (tkey, _key_order(eid))  # `ft` (the edge table) sorts before `fk` (the edge record key)
            s, d = self.idx[src], self.idx[dst]
            if direction == "out":
                adj[s].append(((1, ek, 0), d, ri))
            elif direction == "in":
                adj[d].append(((0, ek, 0), s, ri))
            elif direction == "both":
                adj[d].append(((0, ek, 0), s, ri))  # edges pointing at d: [source, d]
                adj[d].append(((0, ek, 1), d, ri))
                adj[s].append(((1, ek, 0), s, ri))  # edges leaving s: [s, target]
                adj[s].append(((1, ek, 1), d, ri))
            else:
                raise ValueError(f"direction {direction!r}: expected 'out', 'in' or 'both'")
        rp, ci, rel = [0], [], []
        for a in adj:
            a.sort()  # (key, target) first: the relation index only breaks ties between identical keys and targets
            ci += [t for _, t, _r in a]
            rel += [r for _, _t, r in a]
            rp.append(len(ci))
        return np.asarray(rp, np.uint64), np.asarray(ci, np.uint32), rel

    def csr(self, edge_table, direction):
        key = (tuple(edge_table) if isinstance(edge_table, list) else edge_table, direction)
        if key not in self._csr:
            rp, ci = self.csr_arrays(edge_table, direction)
            self._csr[key] = CsrGraph(self.ctx, rp, ci)
        return self._csr[key]

    def expand_snapshot(self, edge_table, direction, frontier, per_source_limit=0):
        """one GraphEdgeScan step over the snapshot of (edge tables, direction) on the GPU"""
        return expand([self.csr(edge_table, direction)], frontier, per_source_limit)

    def ids(self, names):
        return np.asarray([self.idx[n] for n in names], np.uint32)

    def to_names(self, arr):
        return [self.names[int(i)] for i in arr]

    def lookup(self, start, hops, limit=0):
        """start: record ids; hops: [(direction 'out'|'in', edge_table), ...] -> record ids (order + duplicates
        as the reference returns them)"""
        return self.to_names(expand([self.csr(tb, d) for d, tb in hops], self.ids(start), limit))

    def collect(self, start, direction, edge_table, min_depth=1, max_depth=0, inclusive=False):
        return self.to_names(collect(self.csr(edge_table, direction), self.ids([start]), min_depth, max_depth, inclusive))

    def recurse(self, start, direction, edge_table, min_depth, max_depth):
        """default recursion: repeat the hop until the bound, a dead end or a fixed point"""
        g = self.csr(edge_table, direction)
        cur = self.ids([start])
        depth = 0
        while depth < max_depth:
            nxt = expand([g], cur)
            depth += 1
            if nxt.size == 0 or (nxt.size == cur.size and np.array_equal(nxt, cur)):
                return self.to_names(cur) if depth > min_depth else None
            cur = nxt
        return self.to_names(cur) if depth >= min_depth else None

    def hop_masks(self, edge_table, direction, edge_pred=None, target_pred=None):
        """what the shim evaluates a hop's WHERE conditions into: (edge mask per CSR position or None, target mask per
        node id or None).  The predicates take a record's fields (a dict with its `id`).  This costs O(E) on the host per
        condition, so on a real table the bitmap is cached or comes from an index."""
        em = tm = None
        if edge_pred is not None:
            em = np.fromiter((bool(edge_pred({**self.edge_props.get(r, {}), "id": r}))
                              for r in self.edge_records(edge_table, direction)), bool)
        if target_pred is not None:
            tm = np.fromiter((bool(target_pred({**self.node_props.get(n, {}), "id": n})) for n in self.names), bool,
                             len(self.names))
        return em, tm

    def lookup_filtered(self, start, hops, limit=0):
        """start: record ids; hops: [(direction, edge_table, edge_pred | None, target_pred | None), ...], i.e.
        `->(edge_table WHERE edge_pred)->(node WHERE target_pred)` -> record ids, order and duplicates as the
        reference returns them"""
        graphs = [self.csr(tb, d) for d, tb, _e, _t in hops]
        masks = [self.hop_masks(tb, d, e, t) for d, tb, e, t in hops]
        return self.to_names(expand_filtered(graphs, masks, self.ids(start), limit))

    def collect_filtered(self, start, direction, edge_table, edge_pred=None, target_pred=None, min_depth=1, max_depth=0,
                         inclusive=False):
        """`.{min..max+collect}->(edge_table WHERE ..)->(node WHERE ..)`: every BFS level is the filtered hop"""
        masks = self.hop_masks(edge_table, direction, edge_pred, target_pred)
        return self.to_names(collect_filtered(self.csr(edge_table, direction), masks, self.ids([start]), min_depth,
                                              max_depth, inclusive))

    def lookup_batch(self, docs, hops, limit=0):
        """LookupPart::evaluate_batch (exec/parts/lookup.rs:96-112): docs = one list of record ids per row; hops =
        [(direction, edge_table), ...] or [(direction, edge_table, edge_pred | None, target_pred | None), ...] ->
        per row its record ids, as lookup / lookup_filtered returns them, from one batch call"""
        graphs = [self.csr(h[1], h[0]) for h in hops]
        filters = None
        if any(len(h) > 2 and (h[2] is not None or h[3] is not None) for h in hops):
            filters = [self.hop_masks(h[1], h[0], h[2], h[3]) if len(h) > 2 else None for h in hops]
        out = expand_batch(graphs, [self.ids(d) for d in docs], limit, filters)
        return [self.to_names(o) for o in out]

    def collect_batch(self, docs, direction, edge_table, edge_pred=None, target_pred=None, min_depth=1, max_depth=0,
                      inclusive=False):
        """`.{min..max+collect}` per row: docs = one list of start record ids per row -> per row its collected record
        ids, as collect / collect_filtered returns them, from one batch call"""
        filt = None
        if edge_pred is not None or target_pred is not None:
            filt = self.hop_masks(edge_table, direction, edge_pred, target_pred)
        out = collect_batch(self.csr(edge_table, direction), [self.ids(d) for d in docs], min_depth, max_depth, inclusive,
                            filt)
        return [self.to_names(o) for o in out]

    def recurse_filtered(self, start, direction, edge_table, edge_pred, target_pred, min_depth, max_depth):
        """default recursion over the filtered hop"""
        g = self.csr(edge_table, direction)
        masks = self.hop_masks(edge_table, direction, edge_pred, target_pred)
        cur = self.ids([start])
        depth = 0
        while depth < max_depth:
            nxt = expand_filtered([g], [masks], cur)
            depth += 1
            if nxt.size == 0 or (nxt.size == cur.size and np.array_equal(nxt, cur)):
                return self.to_names(cur) if depth > min_depth else None
            cur = nxt
        return self.to_names(cur) if depth >= min_depth else None


class GraphEdgeScan:
    """Mirror of the reference operator (exec/operators/scan/graph.rs:89-147):
    `GraphEdgeScan::new(input, direction, edge_tables, output_mode, version)` + `.with_limit(n)`, `name()`, `attrs()`,
    `execute()`.  `input` yields the source record ids (what the child operator streams); the result is the target
    record id of every matching edge pointer, per source in KV key order, duplicates kept -- served by one
    sdb_graph_expand over the CSR snapshot of (direction, edge tables).  Range bounds on an edge table, `version`
    (time travel) and output modes other than TargetId are the cases INTEGRATION.md leaves on the KV path."""

    DIRECTIONS = {"->": "out", "<-": "in", "<->": "both"}

    def __init__(self, input, direction, edge_tables, output_mode="TargetId", version=None, store=None):
        if direction not in self.DIRECTIONS:
            raise L.SdbError(L.SDB_EUNSUPPORTED, f"direction {direction!r} is not served by the GPU snapshot")
        if output_mode != "TargetId" or version is not None:
            raise L.SdbError(L.SDB_EUNSUPPORTED, "only GraphScanOutput::TargetId without VERSION is served by the GPU snapshot")
        self.input, self.direction, self.edge_tables = input, direction, list(edge_tables)
        self.output_mode, self.version, self.limit, self.store = output_mode, version, None, store

    def with_limit(self, limit):
        self.limit = int(limit)
        return self

    def name(self):
        return "GraphEdgeScan"

    def attrs(self):
        a = [("direction", self.direction), ("tables", ", ".join(self.edge_tables) if self.edge_tables else "*"),
             ("output", self.output_mode)]
        if self.limit is not None:
            a.append(("limit", str(self.limit)))
        return a

    def _snapshot(self):
        tables = None if not self.edge_tables else (self.edge_tables[0] if len(self.edge_tables) == 1 else tuple(self.edge_tables))
        return tables, self.DIRECTIONS[self.direction]

    def execute(self):
        tables, d = self._snapshot()
        sources = list(self.input)
        unknown = [s for s in sources if s not in self.store.idx]  # a record without edges has no graph keys: no output
        frontier = self.store.ids([s for s in sources if s in self.store.idx])
        del unknown
        if self.limit == 0:
            # with_limit(0): the per-source key stream is opened with limit Some(0) and yields nothing
            # (scan/graph.rs:238 -> kvs/scanner.rs:160-172: ScanLimit::Count(min(batch, 0))); None = unlimited
            return []
        return self.store.to_names(self.store.expand_snapshot(tables, d, frontier, self.limit or 0))

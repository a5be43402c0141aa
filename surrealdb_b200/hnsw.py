"""Host-side mirror of the HNSW search path on top of the C ABI.

  HnswIndex.load(...)                 what the Rust shim hands over after HnswFlavor::check_state
                                      (idx/trees/hnsw/mod.rs:187-224): element vectors + per-layer adjacency
  HnswIndex.search_graph(q, k, ef)    Hnsw::knn_search (hnsw/mod.rs:459-482) -> [(dist, element)] ascending
  HnswIndex.search_graph_filtered(..) Hnsw::knn_search_with_filter with one element bitmap per query, any selectivity
  HnswIndex.knn_search(q, k, ef)      HnswIndex::knn_search (hnsw/index.rs:270-335): pending updates first
                                      (search_pendings, :372-420), then the graph with the pending-docs bitmap,
                                      element -> docs expansion through KnnResultBuilder semantics
                                      (idx/trees/knn.rs:363-437): final order (distance, VectorId), <= k
  HnswIndex.add_pending(...)          the Hp log (VectorPendingUpdate, hnsw/mod.rs:88-113) as the Rust shim streams it
  HnswIndex.check_state(state)        Hnsw::check_state (hnsw/mod.rs:187-224): is the device copy still current?
"""
import ctypes as C

import numpy as np

from . import _lib as L

# numpy element type of each sdb_vector_type (VectorType of the index definition)
VT_DTYPE = {"F64": np.float64, "F32": np.float32, "I64": np.int64, "I32": np.int32, "I16": np.int16}


def _int_of(x, vector_type, info):
    """one Number -> the integer type (val/number.rs:136-166, num-traits' ToPrimitive): an integer must fit, a float is
    truncated toward zero and must then fit (NaN and infinities never do)"""
    if isinstance(x, (int, np.integer)) and not isinstance(x, bool):
        v = int(x)
    else:
        f = float(x)
        if f != f or f in (float("inf"), float("-inf")):
            raise L.SdbError(L.SDB_EINVAL, f"{f} cannot be converted to {vector_type}")
        v = int(f)  # truncation toward zero
    if not info.min <= v <= info.max:
        raise L.SdbError(L.SDB_EINVAL, f"{x} is out of the range of {vector_type}")
    return v


def to_vector_type(values, vector_type):
    """Vector::try_from_vector (hnsw/index.rs:286, vector.rs:592-621): the numbers of a query, element or pending vector
    as the index's vector type.  F32 / F64: a float conversion (np.float32 / np.float64).  Integer types: an integer
    keeps its value and must fit; a float is truncated toward zero; anything out of range, or NaN, raises
    SdbError(SDB_EINVAL)."""
    vt = vector_type.upper()
    dt = np.dtype(VT_DTYPE[vt])
    if dt.kind == "f":
        return np.ascontiguousarray(values, dt)
    info = np.iinfo(dt)
    a = np.asarray(values)
    if a.dtype.kind in "iu":  # exact, range-checked without a float round trip (an I64 above 2^53 survives)
        if a.size and (int(a.min()) < info.min or int(a.max()) > info.max):
            raise L.SdbError(L.SDB_EINVAL, f"a value is out of the range of {vt}")
        return np.ascontiguousarray(a.astype(dt))
    if a.dtype.kind == "O":
        flat = [_int_of(x, vt, info) for x in a.ravel().tolist()]
        return np.array(flat, dt).reshape(a.shape)
    f = a.astype(np.float64)
    t = np.trunc(f)
    lim = float(2 ** (8 * dt.itemsize - 1))
    if not np.all(np.isfinite(t) & (t >= -lim) & (t < lim)):
        raise L.SdbError(L.SDB_EINVAL, f"a value is NaN or out of the range of {vt}")
    return np.ascontiguousarray(t.astype(dt))


def _float_key(d):
    """FloatKey's total_cmp order for a non-NaN distance: Python's float comparison ties -0.0 with 0.0, FloatKey puts
    -0.0 first"""
    return d, 0 if d == 0 and np.signbit(d) else 1


class KnnResultBuilder:
    """idx/trees/knn.rs:363-437: a BTreeSet<(FloatKey(dist), VectorId)> capped at knn entries."""

    def __init__(self, knn, vid_key):
        self.knn, self.vid_key, self.items = int(knn), vid_key, []  # items: sorted [(dist, key(vid), vid)]

    def check_add(self, dist):  # accept unless the list is full and the distance is farther than the last
        return not (len(self.items) >= self.knn and self.items and dist > self.items[-1][0])

    def add_vector_id_result(self, dist, vid):
        ent = (dist, self.vid_key(vid), vid)
        # a set: an equal pair collapses
        if not any(_float_key(e[0]) == _float_key(ent[0]) and e[1] == ent[1] for e in self.items):
            self.items.append(ent)
            self.items.sort(key=lambda e: (_float_key(e[0]), e[1]))
        if len(self.items) > self.knn:
            self.items.pop()

    def collect(self):
        return [(d, vid) for d, _, vid in self.items]


class HnswIndex:
    def __init__(self, ctx, vectors, layers, entry_point, metric="EUCLIDEAN", elem_docs=None, minkowski_order=3.0,
                 vector_type="F32"):
        """vectors (n, dim), converted to the vector type; layers = [(row_ptr u64[n+1], col_idx u32[e]), ...] layer 0
        first; elem_docs: optional list of doc-id lists per element (identical vectors share one element:
        hnsw/docs.rs:161-176); default = one doc per element with the same id.  metric: any Distance
        (DIST ... of the index definition); minkowski_order: p of Distance::Minkowski(p), used by MINKOWSKI only;
        vector_type: TYPE ... of the index definition (F64, F32, I64, I32, I16), the arithmetic of every distance."""
        self.vector_type = vector_type.upper()
        if self.vector_type not in L.VTYPE:
            raise L.SdbError(L.SDB_EINVAL, f"unknown vector type {vector_type!r}")
        vec = to_vector_type(vectors, self.vector_type)
        self.n, self.dim = vec.shape
        self.ctx, self.metric = ctx, metric.upper()
        self.elem_docs = elem_docs
        self.pendings = []
        self.versions = None
        nl = len(layers)
        rps = [np.ascontiguousarray(l[0], np.uint64) for l in layers]
        cis = [np.ascontiguousarray(l[1] if len(l[1]) else np.zeros(1, np.uint32), np.uint32) for l in layers]
        RP = (C.c_void_p * nl)(*[a.ctypes.data for a in rps])
        CI = (C.c_void_p * nl)(*[a.ctypes.data for a in cis])
        self.h = C.c_void_p()
        L.check(L.lib().sdb_hnsw_load_typed(ctx.h, self.dim, L.METRIC[self.metric], L.VTYPE[self.vector_type], self.n,
                                            C.c_void_p(vec.ctypes.data), nl, RP, CI, int(entry_point), C.byref(self.h)))
        self._set_order(minkowski_order)

    def _set_order(self, minkowski_order):
        if self.metric == "MINKOWSKI":
            L.check(L.lib().sdb_hnsw_set_minkowski_order(self.h, float(minkowski_order)))

    @classmethod
    def from_device(cls, ctx, x_dev, layers_dev, entry_point, metric="EUCLIDEAN", elem_docs=None, minkowski_order=3.0,
                    vector_type="F32"):
        """wraps device-resident vectors and CSR layers WITHOUT copying them (sdb_hnsw_load_device_typed): x_dev is a torch
        CUDA (n, dim) tensor of the vector type's dtype (F64 float64, F32 float32, I64 int64, I32 int32, I16 int16),
        layers_dev = [(row_ptr int64 (n+1), col_idx int32)] layer 0 first.  The tensors must stay alive (they are kept on
        the object)."""
        self = cls.__new__(cls)
        self.ctx, self.metric, self.elem_docs, self.vector_type = ctx, metric.upper(), elem_docs, vector_type.upper()
        if self.vector_type not in L.VTYPE:
            raise L.SdbError(L.SDB_EINVAL, f"unknown vector type {vector_type!r}")
        if np.dtype(str(x_dev.dtype).replace("torch.", "")) != np.dtype(VT_DTYPE[self.vector_type]):
            raise L.SdbError(L.SDB_EINVAL, f"{x_dev.dtype} vectors for an index of type {self.vector_type}")
        self.n, self.dim = int(x_dev.shape[0]), int(x_dev.shape[1])
        self.pendings, self.versions = [], None
        self._keep = (x_dev, layers_dev)
        nl = len(layers_dev)
        RP = (C.c_void_p * nl)(*[t[0].data_ptr() for t in layers_dev])
        CI = (C.c_void_p * nl)(*[t[1].data_ptr() for t in layers_dev])
        self.h = C.c_void_p()
        L.check(L.lib().sdb_hnsw_load_device_typed(ctx.h, self.dim, L.METRIC[self.metric], L.VTYPE[self.vector_type], self.n,
                                                   C.c_void_p(x_dev.data_ptr()), nl, RP, CI, int(entry_point), C.byref(self.h)))
        self._set_order(minkowski_order)
        return self

    @classmethod
    def from_kv(cls, ctx, dim, state_value, he_items, hn_items_per_layer, metric="EUCLIDEAN", elem_docs=None,
                minkowski_order=3.0, vector_type="F32"):
        """Loads the index straight from raw KV values (staging.py): `state_value` = the Hs value, `he_items` =
        [(element id, He value)], `hn_items_per_layer[l]` = [(node id, Hn value)] of layer l (0 first), each in key
        order.  Decoding happens on the GPU (sdb_hnsw_load_staged, sdb_hnsw_load_staged_typed for the other vector
        types: there an He value of another type counts in n_bad).  Mirrors Hnsw::check_state + HnswLayer::load
        (hnsw/mod.rs:187-224, hnsw/layer.rs:505-560) for indexes without legacy Hl chunks."""
        from . import staging as S
        st = S.parse_hnsw_state(state_value)
        if st["layer0"]["chunks"] or any(l["chunks"] for l in st["layers"]):
            raise L.SdbError(L.SDB_EUNSUPPORTED, "legacy Hl chunks present: run the reference's migration first")
        nl = 1 + len(st["layers"])
        if len(hn_items_per_layer) != nl:
            raise L.SdbError(L.SDB_EINVAL, f"state names {nl} layers, {len(hn_items_per_layer)} given")
        self = cls.__new__(cls)
        self.ctx, self.metric, self.dim, self.elem_docs = ctx, metric.upper(), int(dim), elem_docs
        self.vector_type = vector_type.upper()
        if self.vector_type not in L.VTYPE:
            raise L.SdbError(L.SDB_EINVAL, f"unknown vector type {vector_type!r}")
        self.pendings = []
        self.versions = [st["layer0"]["version"]] + [l["version"] for l in st["layers"]]
        self.n = int(st["next_element_id"])
        vb, vo, vi = S.pack_values(he_items)
        packs = [S.pack_values(it) for it in hn_items_per_layer]
        NB = (C.c_void_p * nl)(*[p[0].ctypes.data for p in packs])
        NO = (C.c_void_p * nl)(*[p[1].ctypes.data for p in packs])
        NI = (C.c_void_p * nl)(*[p[2].ctypes.data for p in packs])
        NN = (C.c_uint64 * nl)(*[len(it) for it in hn_items_per_layer])
        self.h = C.c_void_p()
        bad = C.c_uint64(0)
        ep = -1 if st["enter_point"] is None else int(st["enter_point"])
        if self.vector_type == "F32":
            L.check(L.lib().sdb_hnsw_load_staged(ctx.h, self.dim, L.METRIC[self.metric], self.n, C.c_void_p(vb.ctypes.data),
                                                 C.c_void_p(vo.ctypes.data), C.c_void_p(vi.ctypes.data), len(he_items), nl,
                                                 NB, NO, NI, NN, ep, C.byref(self.h), C.byref(bad)))
        else:
            L.check(L.lib().sdb_hnsw_load_staged_typed(ctx.h, self.dim, L.METRIC[self.metric], L.VTYPE[self.vector_type],
                                                       self.n, C.c_void_p(vb.ctypes.data), C.c_void_p(vo.ctypes.data),
                                                       C.c_void_p(vi.ctypes.data), len(he_items), nl, NB, NO, NI, NN, ep,
                                                       C.byref(self.h), C.byref(bad)))
        self.n_bad = bad.value
        self._set_order(minkowski_order)
        return self

    # ---- freshness: layer versions (Hs) and the pending log (Hp) ---------------------------------------------------
    def check_state(self, state_value):
        """Hnsw::check_state (hnsw/mod.rs:187-224): the persisted HnswState carries one version per layer; a layer
        whose version differs from the loaded one must be reloaded.  Returns True when the device copy is current,
        False when the caller has to rebuild it (HnswIndex.from_kv) before searching."""
        from . import staging as S
        st = S.parse_hnsw_state(state_value)
        cur = [st["layer0"]["version"]] + [l["version"] for l in st["layers"]]
        return self.versions is not None and cur == self.versions and int(st["next_element_id"]) == self.n

    def add_pending(self, vector_id, old_vectors, new_vectors):
        """one VectorPendingUpdate of the Hp range, in key order (hnsw/index.rs:424-452).  vector_id: an int (VectorId::
        DocId) or any other hashable (VectorId::RecordKey); new_vectors empty = deletion."""
        self.pendings.append((vector_id, [to_vector_type(v, self.vector_type) for v in old_vectors],
                              [to_vector_type(v, self.vector_type) for v in new_vectors]))

    def clear_pendings(self):
        """index_pendings applied the log (hnsw/index.rs:138-211): the caller reloads the graph and drops the log"""
        self.pendings = []

    @staticmethod
    def _vid_key(vid):
        """VectorId ordering (derive(PartialOrd, Ord), hnsw/mod.rs:109-113): every DocId sorts before every RecordKey"""
        return (0, int(vid)) if isinstance(vid, (int, np.integer)) else (1, vid)

    def _typed_distances(self, query, vectors):
        """Distance::calculate(&search.pt, &vector) with the index's metric, vector type and Minkowski order, on the
        GPU (sdb_hnsw_distance)"""
        q = to_vector_type(query, self.vector_type)
        v = to_vector_type(vectors, self.vector_type).reshape(-1, self.dim)
        out = np.zeros(v.shape[0], np.float64)
        L.check(L.lib().sdb_hnsw_distance(self.h, C.c_void_p(q.ctypes.data), C.c_void_p(v.ctypes.data), v.shape[0],
                                          C.c_void_p(out.ctypes.data)))
        return out

    def _queries(self, queries):
        """queries as a contiguous (nq, dim) array of the index's vector type (to_vector_type)"""
        q = to_vector_type(queries, self.vector_type)
        if q.ndim == 1:
            q = q[None, :]
        if q.shape[1] != self.dim:  # Error::InvalidVectorDimension  idx/trees/vector.rs:643-652
            raise L.SdbError(L.SDB_EDIM, f"Incorrect vector dimension ({q.shape[1]}). Expected a vector of {self.dim} dimension.")
        return q

    @staticmethod
    def _outputs(nq, k):
        """host outputs of a search: ids, distances, counts, counters"""
        return (np.zeros((nq, max(k, 1)), np.uint64), np.zeros((nq, max(k, 1)), np.float64), np.zeros(nq, np.uint32),
                np.zeros((nq, 2), np.uint64))

    def _pending_mask(self, all_docs_pending):
        m = np.ascontiguousarray(all_docs_pending, np.uint8)
        if m.shape != (self.n,):
            raise L.SdbError(L.SDB_EINVAL, f"pending mask must have one byte per element ({self.n})")
        return m

    def search_graph(self, queries, k, ef, counters=False, truthy=None, all_docs_pending=None):
        """truthy: optional predicate mask, one byte per element (Hnsw::knn_search_with_filter, hnsw/mod.rs:488-515).
        all_docs_pending: optional mask, one byte per element: every document of the element has a pending update
        (the pending_docs argument of Hnsw::knn_search evaluated per element, hnsw/layer.rs:209,320-339).
        queries are converted to the index's vector type (to_vector_type)."""
        q = self._queries(queries)
        nq = q.shape[0]
        ids, dist, cnt, ctr = self._outputs(nq, k)
        if truthy is not None and all_docs_pending is not None:
            # add_if_truthy ignores an element whose documents are all pending (layer.rs:287-296)
            truthy = np.asarray(truthy, np.uint8) & (np.asarray(all_docs_pending, np.uint8) == 0)
        elif all_docs_pending is not None:
            m = self._pending_mask(all_docs_pending)
            L.check(L.lib().sdb_hnsw_search_pending(self.h, C.c_void_p(q.ctypes.data), nq, int(k), int(ef),
                                                    C.c_void_p(m.ctypes.data), C.c_void_p(ids.ctypes.data),
                                                    C.c_void_p(dist.ctypes.data), C.c_void_p(cnt.ctypes.data),
                                                    C.c_void_p(ctr.ctypes.data)))
            return (ids, dist, cnt, ctr) if counters else (ids, dist, cnt)
        if truthy is not None:
            t = np.ascontiguousarray(truthy, np.uint8)
            if t.shape != (self.n,):
                raise L.SdbError(L.SDB_EINVAL, f"predicate mask must have one byte per element ({self.n})")
            L.check(L.lib().sdb_hnsw_search_filtered(self.h, C.c_void_p(q.ctypes.data), nq, int(k), int(ef),
                                                     C.c_void_p(t.ctypes.data), C.c_void_p(ids.ctypes.data),
                                                     C.c_void_p(dist.ctypes.data), C.c_void_p(cnt.ctypes.data),
                                                     C.c_void_p(ctr.ctypes.data)))
        else:
            L.check(L.lib().sdb_hnsw_search(self.h, C.c_void_p(q.ctypes.data), nq, int(k), int(ef),
                                            C.c_void_p(ids.ctypes.data), C.c_void_p(dist.ctypes.data),
                                            C.c_void_p(cnt.ctypes.data), C.c_void_p(ctr.ctypes.data)))
        if counters:
            return ids, dist, cnt, ctr
        return ids, dist, cnt

    def filter_words(self, filters):
        """bool masks (n,) or (n_filters, n) over the elements, or their packed uint32 words (engine.pack_row_filter)
        -> contiguous (n_filters, ceil(n / 32)) uint32 words"""
        from .engine import _filter_args, pack_row_filter
        f = np.asarray(filters)
        if f.dtype == np.bool_:
            if f.shape[-1] != self.n:
                raise L.SdbError(L.SDB_EINVAL, f"filter masks must have one entry per element ({self.n})")
            f = pack_row_filter(f)
        return _filter_args(f, None, 0, self.n)[0]

    def search_graph_filtered(self, queries, k, ef, filters, query_filter=None, counters=False):
        """Hnsw::knn_search_with_filter for a batch whose queries each pick one of several predicates
        (sdb_hnsw_search_filtered_batch): filters = bool masks (n,) / (n_filters, n) or packed uint32 words
        (filter_words); query_filter = one filter index per query (None: filter 0 for every query).  Any selectivity
        is served on the GPU: queries that outgrow the on-chip candidate window finish in the spill tier."""
        from .engine import _query_filter
        q = self._queries(queries)
        nq = q.shape[0]
        f = self.filter_words(filters)
        qf = _query_filter(query_filter, nq)
        ids, dist, cnt, ctr = self._outputs(nq, k)
        L.check(L.lib().sdb_hnsw_search_filtered_batch(self.h, C.c_void_p(q.ctypes.data), nq, int(k), int(ef),
                                                       C.c_void_p(f.ctypes.data), f.shape[0],
                                                       None if qf is None else C.c_void_p(qf.ctypes.data),
                                                       C.c_void_p(ids.ctypes.data), C.c_void_p(dist.ctypes.data),
                                                       C.c_void_p(cnt.ctypes.data), C.c_void_p(ctr.ctypes.data)))
        return (ids, dist, cnt, ctr) if counters else (ids, dist, cnt)

    def last_spilled(self):
        """queries of the last search_graph_filtered call (or waited filtered ticket) that the spill tier finished"""
        return int(L.lib().sdb_hnsw_last_spilled(self.h))

    # ---- asynchronous search: up to 4 tickets in flight per index, completed by wait() in any order -----------------
    def submit_graph(self, queries, k, ef, counters=False, all_docs_pending=None):
        """search_graph (without truthy) queued without a host synchronisation (sdb_hnsw_submit): -> a ticket, whose
        wait() returns what search_graph would have returned"""
        q = self._queries(queries)
        nq = q.shape[0]
        m = None if all_docs_pending is None else self._pending_mask(all_docs_pending)
        out = self._outputs(nq, k)
        ids, dist, cnt, ctr = out
        t = C.c_uint32()
        L.check(L.lib().sdb_hnsw_submit(self.h, C.c_void_p(q.ctypes.data), nq, int(k), int(ef),
                                        None if m is None else C.c_void_p(m.ctypes.data), C.c_void_p(ids.ctypes.data),
                                        C.c_void_p(dist.ctypes.data), C.c_void_p(cnt.ctypes.data),
                                        C.c_void_p(ctr.ctypes.data), C.byref(t)))
        self._tickets()[t.value] = ((q, m) + out, counters)
        return t.value

    def submit_graph_filtered(self, queries, k, ef, filters, query_filter=None, counters=False):
        """search_graph_filtered queued without a host synchronisation (sdb_hnsw_submit_filtered): -> a ticket, whose
        wait() returns what search_graph_filtered would have returned"""
        from .engine import _query_filter
        q = self._queries(queries)
        nq = q.shape[0]
        f = self.filter_words(filters)
        qf = _query_filter(query_filter, nq)
        out = self._outputs(nq, k)
        ids, dist, cnt, ctr = out
        t = C.c_uint32()
        L.check(L.lib().sdb_hnsw_submit_filtered(self.h, C.c_void_p(q.ctypes.data), nq, int(k), int(ef),
                                                 C.c_void_p(f.ctypes.data), f.shape[0],
                                                 None if qf is None else C.c_void_p(qf.ctypes.data),
                                                 C.c_void_p(ids.ctypes.data), C.c_void_p(dist.ctypes.data),
                                                 C.c_void_p(cnt.ctypes.data), C.c_void_p(ctr.ctypes.data), C.byref(t)))
        self._tickets()[t.value] = ((q, f) + out, counters)
        return t.value

    def submit_device(self, d_queries, nq, k, ef, d_out_elems, d_out_dist, d_out_count, d_out_counters=None):
        """sdb_hnsw_submit_device: device pointers (ints), valid until wait(ticket), which then returns None"""
        t = C.c_uint32()
        L.check(L.lib().sdb_hnsw_submit_device(self.h, C.c_void_p(d_queries), int(nq), int(k), int(ef),
                                               C.c_void_p(d_out_elems), C.c_void_p(d_out_dist), C.c_void_p(d_out_count),
                                               C.c_void_p(d_out_counters), C.byref(t)))
        return t.value

    def submit_filtered_device(self, d_queries, nq, k, ef, d_filters, n_filters, query_filter, d_out_elems, d_out_dist,
                               d_out_count, d_out_counters=None):
        """sdb_hnsw_submit_filtered_device: device pointers (ints) valid, and d_filters unchanged, until wait(ticket),
        which then returns None; query_filter is a host array (or None), copied before the call returns"""
        from .engine import _query_filter
        qf = _query_filter(query_filter, nq)
        t = C.c_uint32()
        L.check(L.lib().sdb_hnsw_submit_filtered_device(self.h, C.c_void_p(d_queries), int(nq), int(k), int(ef),
                                                        C.c_void_p(d_filters), int(n_filters),
                                                        None if qf is None else C.c_void_p(qf.ctypes.data),
                                                        C.c_void_p(d_out_elems), C.c_void_p(d_out_dist),
                                                        C.c_void_p(d_out_count), C.c_void_p(d_out_counters), C.byref(t)))
        return t.value

    def wait(self, ticket):
        """completes a ticket (sdb_hnsw_wait): the tuple search_graph / search_graph_filtered would have returned for a
        ticket of submit_graph / submit_graph_filtered, None for the raw device submits.  The ticket is released (and
        its arrays with it) whether or not the wait succeeds."""
        kept = self._tickets().pop(int(ticket), None)
        L.check(L.lib().sdb_hnsw_wait(self.h, int(ticket)))
        if kept is None:
            return None
        (_, _, ids, dist, cnt, ctr), counters = kept
        return (ids, dist, cnt, ctr) if counters else (ids, dist, cnt)

    def _tickets(self):
        """ticket -> the arrays the library reads or writes until its wait (and whether it reports counters)"""
        if not hasattr(self, "_inflight"):
            self._inflight = {}
        return self._inflight

    def knn_search(self, query, k, ef, truthy_docs=None):
        """-> [(vector id, distance)] ordered by (distance, VectorId), at most k  (one query).  Mirrors
        HnswIndex::knn_search (hnsw/index.rs:270-335):
          1. search_pendings (:372-420): the Hp log is folded per VectorId (a later deletion removes it, a later
             update replaces it); every surviving new vector is ranked with Distance::calculate and offered to the
             KnnResultBuilder; the DocIds seen in ANY pending update form the pending_docs bitmap.
          2. search_graph (:341-364) with that bitmap: an element whose docs are all pending is kept in w but not
             expanded (unfiltered) / ignored by add_if_truthy (filtered); add_graph_results adds ALL docs of each
             neighbour (:454-475).
        truthy_docs: optional set of vector ids passing the WHERE condition (cond_filter): an element enters the result
        window if ANY of its docs is truthy (HnswTruthyDocumentFilter::check_any_doc_truthy, hnsw/filter.rs:52-62); a
        pending vector is skipped unless its id is truthy (check_vector_id_truthy).  The executor re-applies the
        WHERE clause downstream."""
        builder = KnnResultBuilder(k, self._vid_key)
        # ---- 1. pendings ----
        all_existing_docs, non_deleted = set(), {}
        for vid, _old, new in self.pendings:
            if isinstance(vid, (int, np.integer)):
                all_existing_docs.add(int(vid))
            if len(new) == 0:
                non_deleted.pop(vid, None)
            else:
                non_deleted[vid] = new
        pending_docs = None
        if all_existing_docs or non_deleted:
            for vid, vectors in non_deleted.items():  # (HashMap iteration order: the builder's set makes it irrelevant)
                if truthy_docs is not None and vid not in truthy_docs:
                    continue
                for d in self._typed_distances(query, np.stack(vectors)):
                    if builder.check_add(float(d)):
                        builder.add_vector_id_result(float(d), vid)
            if all_existing_docs:
                pending_docs = all_existing_docs
        # ---- 2. graph ----
        docs_of = (lambda e: [e]) if self.elem_docs is None else (lambda e: self.elem_docs[e])
        truthy = None
        if truthy_docs is not None:
            truthy = np.zeros(self.n, np.uint8)
            for e in range(self.n):
                truthy[e] = any(d in truthy_docs for d in docs_of(e))
        all_pending = None
        if pending_docs:
            all_pending = np.zeros(self.n, np.uint8)
            for e in range(self.n):
                dl = docs_of(e)
                all_pending[e] = all(int(d) in pending_docs for d in dl)  # an element without docs counts as pending
        q = to_vector_type(query, self.vector_type)[None, :]
        if truthy is not None:  # any selectivity on the GPU; add_if_truthy ignores all-pending elements (layer.rs:287-296)
            if all_pending is not None:
                truthy &= all_pending == 0
            ids, dist, cnt = self.search_graph_filtered(q, k, ef, truthy.astype(bool))
        else:
            ids, dist, cnt = self.search_graph(q, k, ef, all_docs_pending=all_pending)
        for j in range(int(cnt[0])):
            d, e = float(dist[0, j]), int(ids[0, j])
            if builder.check_add(d):
                for doc in docs_of(e):
                    builder.add_vector_id_result(d, int(doc))
        return [(vid, d) for d, vid in builder.collect()]

    def close(self):
        if self.h:
            L.lib().sdb_hnsw_destroy(self.h)  # waits for the tickets in flight: their arrays go after it
            self.h = C.c_void_p()
            self._tickets().clear()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

"""Host-side mirror of the reference's operator interface for the hot path.

The reference is Rust (no cargo/rustc in this image), so the operator glue a maintainer would add behind
a `gpu-knn` cargo feature (INTEGRATION.md) is mirrored here in Python with the same names, argument
meaning and error behaviour, on top of the same C ABI:

  KnnTopK(input, field, query_vector, k, distance)   core/exec/operators/knn_topk.rs:100-118
      .execute()  -> records nearest-first           knn_topk.rs:166-267
      .name() / .attrs()                              knn_topk.rs:133-144   (EXPLAIN output)
  KnnScan(index, vector, k, ef, table_name, ...)      core/exec/operators/scan/knn.rs:68-118,135-347 (HNSW-backed)
  KnnContext: record id -> distance hand-back         core/exec/function/index.rs:289-314
  SortTopK(input, field, fn, query_vector, limit, direction)   core/exec/operators/sort/topk.rs:100-118
      Compute(vector::<fn>(field, $q)) + SortTopK with that single ORDER BY key (planner/select.rs:782-789)
      .execute()  -> records best first, each with the computed value under `alias`

Records are dicts with an "id"; `input` is any iterable yielding them in scan (record-key) order, i.e.
what TableScan yields.

  TableScan(table, records, version) / Union(*inputs) / Filter(input, predicate)
      the sources of `WHERE emb <|k|> $q AND cond`, planned as KnnTopK(Filter(TableScan))
      (exec/planner/select.rs:1642-1652).  KnnTopK over a Filter ranks the source's column with the predicate's
      row bitmap (sdb_knn_bruteforce_filtered) and keeps that column cached per (tables, table versions), so
      statements with different predicates share one staged column (INTEGRATION.md section 8).
"""
import numpy as np

from .engine import Context, VectorColumn, pack_row_filter


class Distance:
    """catalog::Distance (catalog/schema/index.rs:247-284); Debug names as printed by EXPLAIN."""
    Cosine = "Cosine"            # int8 / bf16 tensor-core screens + exact re-rank
    Euclidean = "Euclidean"      # bf16 tensor-core screen + exact re-rank
    Manhattan = "Manhattan"      # this and Chebyshev: the f32 L1 / L-infinity screen + exact re-rank
    Chebyshev = "Chebyshev"
    Hamming = "Hamming"          # exact mismatch counts batched over the queries (k <= 256); k > 256: exact kernel
    Pearson = "Pearson"          # the cosine screens on the centred rows + exact re-rank
    Minkowski = "Minkowski"      # order via VectorColumn.set_minkowski_order: integer orders 1-8 on the f32 Lp screen
                                 # + exact re-rank, every other order on the exact kernel (pow(): ~1e-14 relative)
    Jaccard = "Jaccard"          # set semantics over the values: exact distinct / shared counts batched over the
                                 # queries (k <= 256); k > 256: exact kernel


class KnnContext(dict):
    """rid -> distance of the last KNN operator (exec/function/index.rs:289-314); backs
    vector::distance::knn()."""

    def insert(self, rid, distance):
        self[rid] = distance


def _pick(value, field):
    """Value::pick for a dotted idiom path; missing parts yield None."""
    cur = value
    for part in field.split("."):
        if not isinstance(cur, dict) or part not in cur:
            return None
        cur = cur[part]
    return cur


def extract_vector(value, field):
    """knn_topk.rs:274-288: Some(vec) only for a non-empty array whose elements are all numbers."""
    arr = _pick(value, field)
    if not isinstance(arr, (list, tuple)) or len(arr) == 0:
        return None
    out = []
    for v in arr:
        if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)):
            return None
        out.append(float(v))
    return out


class TableScan:
    """The records of one table in scan (record-key) order.  `version` changes whenever the table does: a staged
    column is reused only for the version it was staged from."""

    def __init__(self, table, records, version=0):
        self.table, self.records, self.version = table, records, version

    def name(self):
        return "TableScan"

    def source_key(self):
        return ("TableScan", self.table), self.version

    def __iter__(self):
        return iter(self.records)


class Union:
    """Several sources one after the other (`FROM a, b`)."""

    def __init__(self, *inputs):
        self.inputs = inputs

    def name(self):
        return "Union"

    def source_key(self):
        keys = [_source_key(i) for i in self.inputs]
        if any(k is None for k in keys):
            return None
        return ("Union",) + tuple(k[0] for k in keys), tuple(k[1] for k in keys)

    def __iter__(self):
        for i in self.inputs:
            yield from i


class Filter:
    """exec Filter operator: the records of `input` for which `predicate(record)` is truthy, in input order."""

    def __init__(self, input, predicate):
        self.input, self.predicate = input, predicate

    def name(self):
        return "Filter"

    def __iter__(self):
        return (rec for rec in self.input if self.predicate(rec))


def _source_key(src):
    """(identity, version) of a cacheable source, None for a plain iterable"""
    fn = getattr(src, "source_key", None)
    return fn() if fn is not None else None


class KnnTopK:
    """Brute-force KNN operator backed by the GPU column.  Pipeline-breaking: consumes the whole input,
    returns the k nearest records ordered by (distance, scan position)."""

    # staged columns of cacheable sources: (source identity, field, dimension, distance) -> (version, column, records).
    # One entry per source and field: a new table version replaces the entry.  Nothing else evicts (the Rust shim owns
    # the column cache and its memory budget, INTEGRATION.md section 8); clear_column_cache() releases everything.
    _column_cache = {}

    def __init__(self, input, field, query_vector, k, distance, ctx=None):
        self.input = input
        self.field = field
        self.query_vector = [float(x) for x in query_vector]
        self.k = int(k)
        self.distance = distance
        self.knn_context = None
        self._ctx = ctx
        self._column = None
        self._records = None

    def with_knn_context(self, knn_context):
        self.knn_context = knn_context
        return self

    def name(self):
        return "KnnTopK"

    def attrs(self):
        return [("field", self.field), ("k", str(self.k)), ("distance", self.distance),
                ("dimension", str(len(self.query_vector)))]

    def _stage(self, source=None):
        """TableScan -> pinned rows -> HBM column (the staging a Rust shim caches per table version)."""
        dim = len(self.query_vector)
        recs, rows, skip = [], [], []
        for rec in (self.input if source is None else source):
            vec = extract_vector(rec, self.field)
            recs.append(rec)
            if vec is None or len(vec) != dim:  # extract_vector None, or compute() Err on dimension mismatch
                rows.append([0.0] * dim)
                skip.append(1)
            else:
                rows.append(vec)
                skip.append(0)
        self._records = recs
        if not recs:
            return None
        arr = np.asarray(rows, np.float64)
        f32 = arr.astype(np.float32)
        dtype = "F32" if np.array_equal(f32.astype(np.float64), arr, equal_nan=True) else "F64"
        if self._ctx is None:
            self._ctx = Context(0)
        col = VectorColumn(self._ctx, dim, self.distance.upper(), dtype, capacity=len(recs))
        col.append(f32 if dtype == "F32" else arr)
        if any(skip):
            col.set_skip(np.asarray(skip, np.uint8))
        col.finalize()
        return col

    def _source_column(self, source):
        """the staged column of `source` (cached per source identity and version when the source has one)"""
        key = _source_key(source)
        if key is None:
            return self._stage(source)
        ident, version = key
        ck = (ident, self.field, len(self.query_vector), self.distance)
        hit = KnnTopK._column_cache.get(ck)
        if hit is not None and hit[0] == version and (self._ctx is None or hit[1].ctx is self._ctx):
            self._records = hit[2]
            return hit[1]
        col = self._stage(source)
        KnnTopK._column_cache[ck] = (version, col, self._records)
        return col

    @classmethod
    def clear_column_cache(cls):
        cls._column_cache.clear()

    def execute(self):
        filt = None
        if self._column is None:
            if isinstance(self.input, Filter):
                # KnnTopK(Filter(source)): rank the source's column with the predicate's row bitmap
                self._column = self._source_column(self.input.input)
            else:
                self._column = self._stage()
        if self._column is None or self.k == 0:
            return []
        q = np.asarray([self.query_vector], np.float64)
        if isinstance(self.input, Filter):
            filt = pack_row_filter([bool(self.input.predicate(rec)) for rec in self._records])
            rows, dist, cnt = self._column.knn(q, self.k, filters=filt)
        else:
            rows, dist, cnt = self._column.knn(q, self.k)
        out = []
        for j in range(int(cnt[0])):
            rec = self._records[int(rows[0, j])]
            if self.knn_context is not None and isinstance(rec, dict) and "id" in rec:
                self.knn_context.insert(rec["id"], float(dist[0, j]))
            out.append(rec)
        return out


# vector functions SortTopK ranks on the GPU: SurrealQL name -> (sdb function name, the metric of the staged column).
# The column's metric only picks its screen copies: vector::similarity::cosine DESC is screened on a COSINE column.
VECTOR_FUNCTIONS = {
    "vector::similarity::cosine": ("SIMILARITY_COSINE", "COSINE"),
    "vector::similarity::pearson": ("PEARSON", "PEARSON"),
    "vector::similarity::jaccard": ("JACCARD", "JACCARD"),
    "vector::dot": ("DOT", "COSINE"),
    "vector::magnitude": ("MAGNITUDE", "COSINE"),
    "vector::distance::euclidean": ("EUCLIDEAN", "EUCLIDEAN"),
    "vector::distance::manhattan": ("MANHATTAN", "MANHATTAN"),
    "vector::distance::chebyshev": ("CHEBYSHEV", "CHEBYSHEV"),
    "vector::distance::hamming": ("HAMMING", "HAMMING"),
}  # (vector::distance::minkowski takes its order as a third argument; a cached column holds one: left to the reference)


class SortTopK(KnnTopK):
    """`SELECT .., vector::<fn>(field, $q) AS alias FROM .. ORDER BY alias ASC|DESC LIMIT k`: the reference plans
    Compute + SortTopK (a heap over Value::compare of the key, earlier rows winning ties) when start + limit <= 1000;
    this operator ranks the staged column with sdb_corpus_order_topk instead, cached like KnnTopK's.  fn is one of
    VECTOR_FUNCTIONS (vector::magnitude takes no query: pass query_vector=None and dim).  A Filter input ranks the
    source's column with the predicate's row bitmap.  The reference raises an error when a ranked row has no vector of
    the query's dimension; this operator does not rank such a statement (SdbError, SDB_EINVAL), the shim leaves it to
    the reference."""

    def __init__(self, input, field, fn, query_vector, limit, direction="ASC", alias=None, order_expr=None,
                 dim=None, ctx=None):
        if fn not in VECTOR_FUNCTIONS:
            from . import _lib as L
            raise L.SdbError(L.SDB_EINVAL, f"SortTopK: {fn} is not ranked on the GPU")
        self.fn, self.direction = fn, direction.upper()
        qv = query_vector if query_vector is not None else [0.0] * int(dim)
        super().__init__(input, field, qv, limit, VECTOR_FUNCTIONS[fn][1], ctx=ctx)
        self.limit, self.alias = int(limit), alias
        self.order_expr = order_expr or (f"{fn}({field})" if query_vector is None else f"{fn}({field}, $q)")
        self._has_query = query_vector is not None

    def name(self):
        return "SortTopK"

    def attrs(self):  # topk.rs:100-118
        return [("order_by", f"{self.order_expr} {self.direction}"), ("limit", str(self.limit))]

    def execute(self):
        from . import _lib as L
        filtered = isinstance(self.input, Filter)
        if self._column is None:
            self._column = self._source_column(self.input.input) if filtered else self._stage()
        if self._column is None or self.limit == 0:
            return []
        dim = len(self.query_vector)
        passes = [bool(self.input.predicate(rec)) for rec in self._records] if filtered else None
        for j, rec in enumerate(self._records):
            vec = extract_vector(rec, self.field)
            if (passes is None or passes[j]) and (vec is None or len(vec) != dim):
                raise L.SdbError(L.SDB_EINVAL, "SortTopK: a ranked row has no vector of the query's dimension "
                                               "(the reference raises an error; not ranked on the GPU)")
        q = np.asarray([self.query_vector], np.float64) if self._has_query else None
        filt = pack_row_filter(passes) if filtered else None
        rows, vals, cnt = self._column.order_topk(q, self.limit, VECTOR_FUNCTIONS[self.fn][0], self.direction,
                                                  filters=filt)
        out = []
        for j in range(int(cnt[0])):
            rec = self._records[int(rows[0, j])]
            out.append(dict(rec, **{self.alias: float(vals[0, j])}) if self.alias else rec)
        return out


class KnnBruteForceLegacy(KnnTopK):
    """The legacy two-pass brute force of the old executor: QueryExecutor::knn (idx/planner/executor.rs:283-311)
    feeds every row's distance to a KnnPriorityList (idx/planner/knn.rs:11-106); the second pass re-iterates the
    table and keeps the rows the list retained, so the result comes back in TABLE order, with the distances served
    by vector::distance::knn() (fnc/vector.rs:79-101) from KnnBruteForceResults::get_dist.

    The retained set is the k nearest; when several rows tie at the k-th distance the reference keeps an arbitrary
    subset of that tie group (`HashSet` iteration order, knn.rs:85-93).  This mirror resolves the tie by scan order
    (a valid outcome of the reference), which makes it the GPU top-k followed by a re-sort on scan position."""

    def name(self):
        return "KnnBruteForce"

    def execute(self):
        if self._column is None:
            self._column = self._stage()
        if self._column is None or self.k == 0:
            return []
        rows, dist, cnt = self._column.knn(np.asarray([self.query_vector], np.float64), self.k)
        n = int(cnt[0])
        order = np.argsort(rows[0, :n], kind="stable")
        out = []
        for j in order:
            rec = self._records[int(rows[0, j])]
            if self.knn_context is not None and isinstance(rec, dict) and "id" in rec:
                self.knn_context.insert(rec["id"], float(dist[0, j]))
            out.append(rec)
        return out


class KnnScan:
    """HNSW-backed KNN scan operator: `WHERE emb <|k,ef|> $q` with an HNSW index (scan/knn.rs:68-118,135-347).
    `index` is the device-resident index (surrealdb_b200.hnsw.HnswIndex) with `.name`; `records` maps a vector id
    (doc id / record key) to the record the scan yields (HnswDocs::get_thing + fetch_and_filter_records_batch).
    residual_cond: optional predicate over records pushed into the search so that rows failing it do not consume top-k
    slots (scan/knn.rs:265-273 -> HnswIndex::knn_search cond_filter)."""

    def __init__(self, index, vector, k, ef, table_name, records, knn_context=None, residual_cond=None,
                 index_name=None, state_value=None):
        self.index, self.vector = index, [float(x) for x in vector]
        self.k, self.ef, self.table_name = int(k), int(ef), table_name
        self.records, self.knn_context, self.residual_cond = records, knn_context, residual_cond
        self.index_name = index_name or getattr(index, "name", "idx")
        self.state_value = state_value

    def name(self):
        return "KnnScan"

    def attrs(self):  # scan/knn.rs:110-117
        return [("index", self.index_name), ("k", str(self.k)), ("ef", str(self.ef)),
                ("dimension", str(len(self.vector)))]

    def cardinality_hint(self):  # CardinalityHint::Bounded(k)
        return ("Bounded", self.k)

    def access_mode(self):
        return "ReadOnly"

    def execute(self):
        from . import _lib as L
        # check_state: the device copy must match the persisted layer versions (scan/knn.rs:258-262)
        if self.state_value is not None and not self.index.check_state(self.state_value):
            raise L.SdbError(L.SDB_EINVAL, "Failed to check HNSW index state: the device copy is stale (reload it)")
        if len(self.vector) != self.index.dim:  # Vector::check_dimension  idx/trees/vector.rs:643-652
            raise L.SdbError(L.SDB_EDIM, f"Incorrect vector dimension ({len(self.vector)}). Expected a vector of "
                                         f"{self.index.dim} dimension.")
        truthy = None
        if self.residual_cond is not None:
            truthy = {vid for vid, rec in self.records.items() if self.residual_cond(rec)}
        res = self.index.knn_search(self.vector, self.k, self.ef, truthy_docs=truthy)
        out = []
        for vid, dist in res:
            rec = self.records.get(vid)
            if rec is None:  # HnswDocs::get_thing returned None: the doc vanished
                continue
            if self.knn_context is not None:
                self.knn_context.insert(rec["id"], dist)
            out.append(rec)
        return out

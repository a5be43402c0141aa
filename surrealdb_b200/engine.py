"""Thin object wrappers over the C ABI handles (sdb_ctx, sdb_corpus)."""
import ctypes as C

import numpy as np

from . import _lib as L


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


def pack_row_filter(mask):
    """bool mask over the corpus rows (or a 2-D stack of masks) -> uint32 words of the filtered KNN bitmaps:
    bit r = bit r % 32 of word r // 32, ceil(rows / 32) words per mask."""
    m = np.asarray(mask, dtype=bool)
    flat = m.reshape(-1, m.shape[-1]) if m.ndim else m.reshape(1, 1)
    n = flat.shape[1]
    words = (n + 31) // 32
    padded = np.zeros((flat.shape[0], words * 32), bool)
    padded[:, :n] = flat
    packed = np.packbits(padded, axis=1, bitorder="little").view("<u4").astype(np.uint32)
    return packed.reshape(m.shape[:-1] + (words,)) if m.ndim else packed[0]


def _filter_args(filters, query_filter, nq, n_rows):
    """(uint32 bitmaps (n_filters, W), uint32 indices (nq,) or None) -- contiguous, ready for the C calls.  The
    library reads W = ceil(n_rows / 32) words per bitmap, so a bitmap of any other width is refused."""
    f = np.ascontiguousarray(filters, np.uint32)
    if f.ndim == 1:
        f = f[None, :]
    if f.ndim != 2 or f.shape[1] != (n_rows + 31) // 32:
        raise L.SdbError(L.SDB_EINVAL, f"filters must be (n_filters, {(n_rows + 31) // 32}) uint32 words for "
                                       f"{n_rows} rows, got {f.shape}")
    return f, _query_filter(query_filter, nq)


def _query_filter(query_filter, nq):
    if query_filter is None:
        return None
    qf = np.ascontiguousarray(query_filter, np.uint32).reshape(-1)
    if qf.size != nq:
        raise L.SdbError(L.SDB_EINVAL, f"query_filter has {qf.size} entries for {nq} queries")
    return qf


class Context:
    """sdb_ctx: one CUDA device."""

    def __init__(self, device=0, _handle=None):
        self.h = C.c_void_p()
        if _handle is not None:
            self.h = C.c_void_p(_handle)
        else:
            L.check(L.lib().sdb_ctx_create(device, C.byref(self.h)))
        self.device = device

    @staticmethod
    def create_multi(devices):
        """one process, several GPUs: contexts sharing one NCCL communicator (sdb_ctx_create_multi)"""
        devs = (C.c_int * len(devices))(*devices)
        out = (C.c_void_p * len(devices))()
        L.check(L.lib().sdb_ctx_create_multi(devs, len(devices), out))
        return [Context(d, _handle=out[i]) for i, d in enumerate(devices)]

    @staticmethod
    def comm_unique_id():
        """128 bytes rank 0 hands to the other ranks (any out-of-band channel) before comm_init_rank"""
        buf = (C.c_uint8 * L.COMM_ID_BYTES)()
        L.check(L.lib().sdb_comm_unique_id(buf))
        return bytes(buf)

    def comm_init_rank(self, nranks, rank, unique_id):
        buf = (C.c_uint8 * L.COMM_ID_BYTES).from_buffer_copy(unique_id)
        L.check(L.lib().sdb_comm_init_rank(self.h, int(nranks), int(rank), buf))

    def comm_size(self):
        return int(L.lib().sdb_comm_size(self.h))

    def stream(self):
        """raw cudaStream_t (int) all kernels of this context run on"""
        return int(L.lib().sdb_ctx_stream(self.h) or 0)

    def cancel(self):
        """raise the context's cancel flag (any thread); running / later calls return SDB_ECANCELLED until cancel_reset"""
        L.lib().sdb_ctx_cancel(self.h)

    def cancel_reset(self):
        L.lib().sdb_ctx_cancel_reset(self.h)

    def kernel_launches(self):
        return int(L.lib().sdb_ctx_kernel_launches(self.h))

    def close(self):
        if self.h:
            L.lib().sdb_ctx_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class VectorColumn:
    """sdb_corpus: device-resident N x D column of one vector field, in scan order."""

    def __init__(self, ctx, dim, metric="COSINE", dtype="F32", capacity=1 << 20):
        self.ctx, self.dim, self.metric, self.dtype = ctx, int(dim), metric.upper(), dtype.upper()
        self.row_base = 0  # global id of row 0 (set_row_base)
        self.h = C.c_void_p()
        L.check(L.lib().sdb_corpus_create(ctx.h, self.dim, L.DTYPE[self.dtype], L.METRIC[self.metric],
                                          int(capacity), C.byref(self.h)))

    def __len__(self):
        return int(L.lib().sdb_corpus_rows(self.h))

    def append(self, rows):
        npdt = np.float32 if self.dtype == "F32" else np.float64
        rows = np.ascontiguousarray(rows, npdt)
        if rows.ndim != 2 or rows.shape[1] != self.dim:
            raise L.SdbError(L.SDB_EDIM, f"rows must be (n, {self.dim})")
        L.check(L.lib().sdb_corpus_append(self.h, _ptr(rows), rows.shape[0]))

    def append_device(self, dev_ptr, n):
        L.check(L.lib().sdb_corpus_append_device(self.h, C.c_void_p(dev_ptr), int(n)))

    def append_synthetic(self, seed, first_row, n):
        L.check(L.lib().sdb_corpus_append_synthetic(self.h, int(seed), int(first_row), int(n)))

    def read_rows(self, first_row, n):
        """rows [first_row, first_row+n) of the device-resident master copy as a numpy array"""
        out = np.empty((int(n), self.dim), np.float32 if self.dtype == "F32" else np.float64)
        L.check(L.lib().sdb_corpus_read_rows(self.h, int(first_row), int(n), _ptr(out)))
        return out

    def set_skip(self, skip):
        if skip is None:
            L.check(L.lib().sdb_corpus_set_skip(self.h, None, 0))
        else:
            s = np.ascontiguousarray(skip, np.uint8)
            L.check(L.lib().sdb_corpus_set_skip(self.h, _ptr(s), s.size))

    def remove(self, row_ids):
        """tombstone rows (scan positions): excluded from every later search, no re-finalize needed"""
        ids = np.ascontiguousarray(row_ids, np.uint64)
        L.check(L.lib().sdb_corpus_remove(self.h, _ptr(ids), ids.size))

    def finalize(self):
        L.check(L.lib().sdb_corpus_finalize(self.h))

    def set_screen(self, name):
        L.check(L.lib().sdb_corpus_set_screen(self.h, L.SCREEN[name.upper()]))

    def set_minkowski_order(self, order):
        L.check(L.lib().sdb_corpus_set_minkowski_order(self.h, float(order)))

    def set_schedule(self, streaming):
        """True (default): streaming tensor-core screen with in-kernel threshold refinement; False: multi-pass"""
        L.check(L.lib().sdb_corpus_set_schedule(self.h, int(bool(streaming))))

    def set_exact(self, exact):
        """False = opt-in approximate mode (no proof, no exact fallback)"""
        L.check(L.lib().sdb_corpus_set_exact(self.h, int(bool(exact))))

    def knn(self, queries, k, cancel_flag=None, filters=None, query_filter=None):
        """queries (nq, dim) float64 -> (rows u64 (nq,k), dist f64 (nq,k), count u32 (nq,)).
        filters: optional uint32 bitmaps (n_filters, ceil(rows/32)) from pack_row_filter; query q then ranks only
        the rows of filters[query_filter[q]] (query_filter None: every query uses filters[0])."""
        q = np.ascontiguousarray(queries, np.float64)
        if q.ndim == 1:
            q = q[None, :]
        if q.shape[1] != self.dim:
            # Error::InvalidVectorDimension analogue; KnnTopK itself never raises it (it skips rows), the
            # HNSW path does (idx/trees/vector.rs:643-652)
            raise L.SdbError(L.SDB_EDIM, f"query dimension {q.shape[1]} != {self.dim}")
        nq = q.shape[0]
        rows = np.zeros((nq, max(k, 1)), np.uint64)
        dist = np.zeros((nq, max(k, 1)), np.float64)
        cnt = np.zeros(nq, np.uint32)
        cf = None if cancel_flag is None else C.c_void_p(cancel_flag.ctypes.data)
        if filters is None:
            L.check(L.lib().sdb_knn_bruteforce(self.h, _ptr(q), nq, int(k), _ptr(rows), _ptr(dist), _ptr(cnt), cf))
        else:
            f, qf = _filter_args(filters, query_filter, nq, len(self))
            L.check(L.lib().sdb_knn_bruteforce_filtered(self.h, _ptr(q), nq, int(k), _ptr(f), f.shape[0],
                                                        None if qf is None else _ptr(qf), _ptr(rows), _ptr(dist),
                                                        _ptr(cnt), cf))
        return rows[:, :k], dist[:, :k], cnt

    def knn_device_filtered(self, d_queries, nq, k, d_filters, n_filters, query_filter, row_base, d_out_rows,
                            d_out_dist, d_out_count):
        """device pointers (ints) for queries, bitmaps and outputs; query_filter is a host array (or None).  d_filters
        must hold n_filters x ceil(len(self) / 32) uint32 words (the library reads exactly that many)."""
        qf = _query_filter(query_filter, nq)
        L.check(L.lib().sdb_knn_bruteforce_filtered_device(self.h, C.c_void_p(d_queries), int(nq), int(k),
                                                           C.c_void_p(d_filters), int(n_filters),
                                                           None if qf is None else _ptr(qf), int(row_base),
                                                           C.c_void_p(d_out_rows), C.c_void_p(d_out_dist),
                                                           C.c_void_p(d_out_count)))

    def knn_device(self, d_queries, nq, k, row_base, d_out_rows, d_out_dist, d_out_count):
        """all arguments are raw device pointers (ints); results complete on return."""
        L.check(L.lib().sdb_knn_bruteforce_device(self.h, C.c_void_p(d_queries), int(nq), int(k), int(row_base),
                                                  C.c_void_p(d_out_rows), C.c_void_p(d_out_dist),
                                                  C.c_void_p(d_out_count)))

    # ---- asynchronous batches (device pointers; buffers must stay valid until wait) ----
    def submit_device(self, d_queries, nq, k, row_base, d_out_rows, d_out_dist, d_out_count):
        t = C.c_uint32()
        L.check(L.lib().sdb_knn_submit_device(self.h, C.c_void_p(d_queries), int(nq), int(k), int(row_base),
                                              C.c_void_p(d_out_rows), C.c_void_p(d_out_dist), C.c_void_p(d_out_count),
                                              C.byref(t)))
        return t.value

    def submit_host(self, h_queries, nq, k, h_out_rows, h_out_dist, h_out_count):
        """raw host pointers (ints), pinned for overlap"""
        t = C.c_uint32()
        L.check(L.lib().sdb_knn_submit(self.h, C.c_void_p(h_queries), int(nq), int(k), C.c_void_p(h_out_rows),
                                       C.c_void_p(h_out_dist), C.c_void_p(h_out_count), C.byref(t)))
        return t.value

    def submit_host_filtered(self, h_queries, nq, k, h_filters, n_filters, query_filter, h_out_rows, h_out_dist,
                             h_out_count):
        """raw host pointers (ints) like submit_host, plus the host bitmaps (valid until wait); query_filter is a host
        array (or None), copied before the call returns.  h_filters must hold n_filters x ceil(len(self) / 32) words."""
        qf = _query_filter(query_filter, nq)
        t = C.c_uint32()
        L.check(L.lib().sdb_knn_submit_filtered(self.h, C.c_void_p(h_queries), int(nq), int(k), C.c_void_p(h_filters),
                                                int(n_filters), None if qf is None else _ptr(qf),
                                                C.c_void_p(h_out_rows), C.c_void_p(h_out_dist),
                                                C.c_void_p(h_out_count), C.byref(t)))
        return t.value

    def submit_device_filtered(self, d_queries, nq, k, d_filters, n_filters, query_filter, row_base, d_out_rows,
                               d_out_dist, d_out_count):
        """asynchronous knn_device_filtered: device pointers (ints) valid until wait; query_filter is a host array (or
        None), copied before the call returns"""
        qf = _query_filter(query_filter, nq)
        t = C.c_uint32()
        L.check(L.lib().sdb_knn_submit_filtered_device(self.h, C.c_void_p(d_queries), int(nq), int(k),
                                                       C.c_void_p(d_filters), int(n_filters),
                                                       None if qf is None else _ptr(qf), int(row_base),
                                                       C.c_void_p(d_out_rows), C.c_void_p(d_out_dist),
                                                       C.c_void_p(d_out_count), C.byref(t)))
        return t.value

    def wait(self, ticket):
        L.check(L.lib().sdb_knn_wait(self.h, int(ticket)))

    # ---- row-sharded search (collective over the context's communicator) ----
    def set_row_base(self, row_base):
        L.check(L.lib().sdb_corpus_set_row_base(self.h, int(row_base)))
        self.row_base = int(row_base)

    def sharded_submit_device(self, d_queries, nq, k, d_out_rows, d_out_dist, d_out_count):
        t = C.c_uint32()
        L.check(L.lib().sdb_knn_sharded_submit_device(self.h, C.c_void_p(d_queries), int(nq), int(k),
                                                      C.c_void_p(d_out_rows), C.c_void_p(d_out_dist),
                                                      C.c_void_p(d_out_count), C.byref(t)))
        return t.value

    def sharded_submit_host(self, h_queries, nq, k, h_out_rows, h_out_dist, h_out_count):
        t = C.c_uint32()
        L.check(L.lib().sdb_knn_sharded_submit(self.h, C.c_void_p(h_queries), int(nq), int(k), C.c_void_p(h_out_rows),
                                               C.c_void_p(h_out_dist), C.c_void_p(h_out_count), C.byref(t)))
        return t.value

    def sharded_submit_filtered_host(self, h_queries, nq, k, h_filters, n_filters, query_filter, n_rows_total,
                                     h_out_rows, h_out_dist, h_out_count):
        """raw host pointers (ints) like sharded_submit_host, plus the host bitmaps over the GLOBAL rows: n_filters x
        ceil(n_rows_total / 32) words, valid until sharded_wait; query_filter is a host array (or None)"""
        qf = _query_filter(query_filter, nq)
        t = C.c_uint32()
        L.check(L.lib().sdb_knn_sharded_submit_filtered(self.h, C.c_void_p(h_queries), int(nq), int(k),
                                                        C.c_void_p(h_filters), int(n_filters),
                                                        None if qf is None else _ptr(qf), int(n_rows_total),
                                                        C.c_void_p(h_out_rows), C.c_void_p(h_out_dist),
                                                        C.c_void_p(h_out_count), C.byref(t)))
        return t.value

    def sharded_submit_filtered_device(self, d_queries, nq, k, d_filters, n_filters, query_filter, n_rows_total,
                                       d_out_rows, d_out_dist, d_out_count):
        """device pointers (ints) like sharded_submit_device, plus the device bitmaps over the GLOBAL rows"""
        qf = _query_filter(query_filter, nq)
        t = C.c_uint32()
        L.check(L.lib().sdb_knn_sharded_submit_filtered_device(self.h, C.c_void_p(d_queries), int(nq), int(k),
                                                               C.c_void_p(d_filters), int(n_filters),
                                                               None if qf is None else _ptr(qf), int(n_rows_total),
                                                               C.c_void_p(d_out_rows), C.c_void_p(d_out_dist),
                                                               C.c_void_p(d_out_count), C.byref(t)))
        return t.value

    def order_sharded_submit_host(self, h_queries, nq, k, fn, order, h_out_rows, h_out_values, h_out_count,
                                  h_filters=None, n_filters=0, query_filter=None, n_rows_total=0):
        """`ORDER BY vector::<fn>(field, $q) ASC|DESC LIMIT k` on a row-sharded column, collective like
        sharded_submit_host: raw host pointers (ints, valid until sharded_wait; h_queries 0 for MAGNITUDE), fn and order
        as in order_topk.  h_filters: optional host bitmaps over the GLOBAL rows (n_filters x ceil(n_rows_total / 32)
        words); query_filter is a host array (or None)."""
        qf = _query_filter(query_filter, nq)
        t = C.c_uint32()
        L.check(L.lib().sdb_corpus_order_sharded_submit(self.h, C.c_void_p(h_queries or None), int(nq),
                                                        self._fn_code(fn), self._order_code(order), int(k),
                                                        C.c_void_p(h_filters or None), int(n_filters),
                                                        None if qf is None else _ptr(qf), int(n_rows_total),
                                                        C.c_void_p(h_out_rows), C.c_void_p(h_out_values),
                                                        C.c_void_p(h_out_count), C.byref(t)))
        return t.value

    def order_sharded_submit_device(self, d_queries, nq, k, fn, order, d_out_rows, d_out_values, d_out_count,
                                    d_filters=None, n_filters=0, query_filter=None, n_rows_total=0):
        """order_sharded_submit_host on device pointers (ints): queries, bitmaps over the GLOBAL rows and outputs"""
        qf = _query_filter(query_filter, nq)
        t = C.c_uint32()
        L.check(L.lib().sdb_corpus_order_sharded_submit_device(self.h, C.c_void_p(d_queries or None), int(nq),
                                                               self._fn_code(fn), self._order_code(order), int(k),
                                                               C.c_void_p(d_filters or None), int(n_filters),
                                                               None if qf is None else _ptr(qf), int(n_rows_total),
                                                               C.c_void_p(d_out_rows), C.c_void_p(d_out_values),
                                                               C.c_void_p(d_out_count), C.byref(t)))
        return t.value

    def sharded_wait(self, ticket):
        L.check(L.lib().sdb_knn_sharded_wait(self.h, int(ticket)))

    def project(self, fn, query=None):
        """One value per row of `vector::<fn>(row, query)` in the reference's f64 arithmetic (fnc/vector.rs): fn is a
        metric name ("EUCLIDEAN", "MANHATTAN", ... = vector::distance::*, "COSINE" = 1 - similarity, "PEARSON" =
        vector::similarity::pearson) or "SIMILARITY_COSINE" / "DOT" / "MAGNITUDE"."""
        code = self._fn_code(fn)
        out = np.zeros(len(self), np.float64)
        q = None
        if query is not None:
            q = np.ascontiguousarray(query, np.float64)
            if q.shape != (self.dim,):  # check_same_dimension  fnc/util/math/vector.rs:23-32
                raise L.SdbError(L.SDB_EDIM, "The two vectors must be of the same dimension.")
        L.check(L.lib().sdb_corpus_project(self.h, _ptr(q) if q is not None else None, code, _ptr(out)))
        return out

    @staticmethod
    def _fn_code(fn):
        """a project() function name, or its integer id as is (unknown ids reach the library, which refuses them)"""
        if isinstance(fn, (int, np.integer)):
            return int(fn)
        fn = fn.upper()
        return L.VECTOR_FN[fn] if fn in L.VECTOR_FN else L.METRIC[fn]

    @staticmethod
    def _order_code(order):
        return int(order) if isinstance(order, (int, np.integer)) else L.ORDER[order.upper()]

    def order_topk(self, queries, k, fn, order, filters=None, query_filter=None):
        """`ORDER BY vector::<fn>(field, $q) ASC|DESC LIMIT k` (SortTopK over project()'s values): fn as in project(),
        order "ASC" / "DESC".  queries (nq, dim) float64, or None for "MAGNITUDE" with nq = 1.  filters / query_filter
        as in knn().  -> (rows u64 (nq,k), values f64 (nq,k), count u32 (nq,))"""
        code = self._fn_code(fn)
        if queries is None:
            q = None
            nq = 1
        else:
            q = np.ascontiguousarray(queries, np.float64)
            if q.ndim == 1:
                q = q[None, :]
            if q.shape[1] != self.dim:  # check_same_dimension  fnc/util/math/vector.rs:23-32
                raise L.SdbError(L.SDB_EDIM, "The two vectors must be of the same dimension.")
            nq = q.shape[0]
        rows = np.zeros((nq, max(k, 1)), np.uint64)
        vals = np.zeros((nq, max(k, 1)), np.float64)
        cnt = np.zeros(nq, np.uint32)
        f, qf = (None, None) if filters is None else _filter_args(filters, query_filter, nq, len(self))
        L.check(L.lib().sdb_corpus_order_topk(self.h, None if q is None else _ptr(q), nq, code, self._order_code(order),
                                              int(k), None if f is None else _ptr(f), 0 if f is None else f.shape[0],
                                              None if qf is None else _ptr(qf), _ptr(rows), _ptr(vals), _ptr(cnt)))
        return rows[:, :k], vals[:, :k], cnt

    def order_topk_device(self, d_queries, nq, k, fn, order, row_base, d_out_rows, d_out_values, d_out_count,
                          d_filters=None, n_filters=0, query_filter=None):
        """order_topk on device pointers (ints; d_queries 0 for MAGNITUDE); query_filter is a host array (or None)"""
        qf = _query_filter(query_filter, nq)
        L.check(L.lib().sdb_corpus_order_topk_device(self.h, C.c_void_p(d_queries or None), int(nq),
                                                     self._fn_code(fn), self._order_code(order), int(k),
                                                     C.c_void_p(d_filters or None), int(n_filters),
                                                     None if qf is None else _ptr(qf), int(row_base),
                                                     C.c_void_p(d_out_rows), C.c_void_p(d_out_values),
                                                     C.c_void_p(d_out_count)))

    def order_submit_host(self, h_queries, nq, k, fn, order, h_out_rows, h_out_values, h_out_count, h_filters=None,
                          n_filters=0, query_filter=None):
        """asynchronous order_topk on raw host pointers (ints, valid until wait), like submit_host_filtered"""
        qf = _query_filter(query_filter, nq)
        t = C.c_uint32()
        L.check(L.lib().sdb_corpus_order_submit(self.h, C.c_void_p(h_queries or None), int(nq), self._fn_code(fn),
                                                self._order_code(order), int(k), C.c_void_p(h_filters or None),
                                                int(n_filters), None if qf is None else _ptr(qf),
                                                C.c_void_p(h_out_rows), C.c_void_p(h_out_values),
                                                C.c_void_p(h_out_count), C.byref(t)))
        return t.value

    def order_submit_device(self, d_queries, nq, k, fn, order, row_base, d_out_rows, d_out_values, d_out_count,
                            d_filters=None, n_filters=0, query_filter=None):
        """asynchronous order_topk_device (device pointers valid until wait)"""
        qf = _query_filter(query_filter, nq)
        t = C.c_uint32()
        L.check(L.lib().sdb_corpus_order_submit_device(self.h, C.c_void_p(d_queries or None), int(nq),
                                                       self._fn_code(fn), self._order_code(order), int(k),
                                                       C.c_void_p(d_filters or None), int(n_filters),
                                                       None if qf is None else _ptr(qf), int(row_base),
                                                       C.c_void_p(d_out_rows), C.c_void_p(d_out_values),
                                                       C.c_void_p(d_out_count), C.byref(t)))
        return t.value

    def stats(self):
        s = L.KnnStats()
        L.check(L.lib().sdb_knn_last_stats(self.h, C.byref(s)))
        return {f[0]: getattr(s, f[0]) for f in L.KnnStats._fields_}

    def close(self):
        if self.h:
            L.lib().sdb_corpus_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def topk_merge_device(ctx, n_lists, nq, k, d_rows, d_dist, d_counts, d_out_rows, d_out_dist, d_out_count,
                      stride_rows=0, stride_dist=0, stride_counts=0):
    L.check(L.lib().sdb_topk_merge_device(ctx.h, n_lists, nq, k, C.c_void_p(d_rows), C.c_void_p(d_dist),
                                          C.c_void_p(d_counts), stride_rows, stride_dist, stride_counts,
                                          C.c_void_p(d_out_rows), C.c_void_p(d_out_dist), C.c_void_p(d_out_count)))


def order_merge_device(ctx, n_lists, nq, k, order, d_rows, d_values, d_counts, d_out_rows, d_out_values, d_out_count,
                       stride_rows=0, stride_values=0, stride_counts=0):
    """topk_merge_device for an ORDER BY ranking: lists and result in (value, row) order for order "ASC" / "DESC"."""
    L.check(L.lib().sdb_order_merge_device(ctx.h, n_lists, nq, k, VectorColumn._order_code(order), C.c_void_p(d_rows),
                                           C.c_void_p(d_values), C.c_void_p(d_counts), stride_rows, stride_values,
                                           stride_counts, C.c_void_p(d_out_rows), C.c_void_p(d_out_values),
                                           C.c_void_p(d_out_count)))


def shard_block_layout(nq, k):
    """byte layout of one rank's result block inside the all-gather buffer:
    rows u64[nq*k] | dist f64[nq*k] | count u32[nq] (padded to 16 bytes)."""
    off_rows, off_dist = 0, nq * k * 8
    off_cnt = 2 * nq * k * 8
    size = (off_cnt + nq * 4 + 15) // 16 * 16
    return off_rows, off_dist, off_cnt, size


def knn_sharded_multi(shards, queries, k, filters=None, query_filter=None, n_rows_total=None):
    """one process, N GPUs: shards[i] is the VectorColumn on the i-th context of Context.create_multi.
    filters: optional uint32 bitmaps (n_filters, ceil(n_rows_total / 32)) over the GLOBAL rows (pack_row_filter of
    global masks), as in VectorColumn.knn; n_rows_total defaults to the largest row_base + len over the shards."""
    q = np.ascontiguousarray(queries, np.float64)
    nq = q.shape[0]
    rows = np.zeros((nq, max(k, 1)), np.uint64)
    dist = np.zeros((nq, max(k, 1)), np.float64)
    cnt = np.zeros(nq, np.uint32)
    hs = (C.c_void_p * len(shards))(*[s.h for s in shards])
    if filters is None:
        L.check(L.lib().sdb_knn_sharded_multi(hs, len(shards), _ptr(q), nq, int(k), _ptr(rows), _ptr(dist), _ptr(cnt)))
    else:
        if n_rows_total is None:
            n_rows_total = max(s.row_base + len(s) for s in shards)
        f, qf = _filter_args(filters, query_filter, nq, int(n_rows_total))
        L.check(L.lib().sdb_knn_sharded_multi_filtered(hs, len(shards), _ptr(q), nq, int(k), _ptr(f), f.shape[0],
                                                       None if qf is None else _ptr(qf), int(n_rows_total),
                                                       _ptr(rows), _ptr(dist), _ptr(cnt)))
    return rows[:, :k], dist[:, :k], cnt


def order_sharded_multi(shards, queries, k, fn, order, filters=None, query_filter=None, n_rows_total=None):
    """`ORDER BY vector::<fn>(field, $q) ASC|DESC LIMIT k` over one process's N GPUs: shards as in knn_sharded_multi,
    fn and order as in VectorColumn.order_topk (queries None for "MAGNITUDE", nq = 1), filters over the GLOBAL rows.
    -> (rows u64 (nq,k), values f64 (nq,k), count u32 (nq,))"""
    if queries is None:
        q, nq = None, 1
    else:
        q = np.ascontiguousarray(queries, np.float64)
        if q.ndim == 1:
            q = q[None, :]
        nq = q.shape[0]
    rows = np.zeros((nq, max(k, 1)), np.uint64)
    vals = np.zeros((nq, max(k, 1)), np.float64)
    cnt = np.zeros(nq, np.uint32)
    hs = (C.c_void_p * len(shards))(*[s.h for s in shards])
    f, qf = None, None
    if filters is not None:
        if n_rows_total is None:
            n_rows_total = max(s.row_base + len(s) for s in shards)
        f, qf = _filter_args(filters, query_filter, nq, int(n_rows_total))
    L.check(L.lib().sdb_corpus_order_sharded_multi(hs, len(shards), None if q is None else _ptr(q), nq,
                                                   VectorColumn._fn_code(fn), VectorColumn._order_code(order), int(k),
                                                   None if f is None else _ptr(f), 0 if f is None else f.shape[0],
                                                   None if qf is None else _ptr(qf), int(n_rows_total or 0),
                                                   _ptr(rows), _ptr(vals), _ptr(cnt)))
    return rows[:, :k], vals[:, :k], cnt

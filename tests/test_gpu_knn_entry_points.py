"""The brute-force KNN entry points held against each other through the C ABI:
  * what each one does with an empty batch and with a cancel flag that is already set;
  * a fifth batch while four tickets are in flight, and a wait on an unknown or already completed ticket;
  * one seeded batch, unfiltered and with two row filters, handed over every way the ABI offers (blocking or ticketed,
    host or device buffers, unsharded or as the only rank of a sharded corpus): the same bytes everywhere, and the
    same kernel launches within the unsharded and within the sharded calls;
  * every handle closed, the library holds no allocation more than before.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, DIM, NQ, K = 20_000, 64, 48, 10
UNSHARDED = ("blocking_host", "blocking_device", "ticket_host", "ticket_device")
SHARDED = ("sharded_host", "sharded_device", "sharded_multi")


def live():
    from surrealdb_b200 import _lib as L
    n, b = C.c_uint64(), C.c_uint64()
    L.lib().sdb_debug_live_allocations(C.byref(n), C.byref(b))
    return n.value, b.value


def launches_of(col):
    return col.stats()["kernel_launches"]


class Batch:
    """one seeded batch: host and device queries, two row filters (one passing half the rows, one few enough for the
    direct regime, so the filtered batch runs permuted) and the filter index of each query"""

    def __init__(self, nq=NQ, seed=5):
        import torch
        from surrealdb_b200.engine import pack_row_filter
        rng = np.random.default_rng(seed)
        self.corpus = rng.uniform(-1, 1, (N, DIM)).astype(np.float32)
        self.nq = nq
        self.q = np.ascontiguousarray(rng.uniform(-1, 1, (nq, DIM)))
        self.dq = torch.from_numpy(self.q).cuda()
        masks = np.zeros((2, N), bool)
        masks[0] = rng.random(N) < 0.5
        masks[1, rng.choice(N, 1500, replace=False)] = True
        self.f = np.ascontiguousarray(pack_row_filter(masks))
        self.df = torch.from_numpy(self.f.view(np.int32)).cuda()
        self.qf = np.ascontiguousarray(np.arange(nq) % 2, np.uint32)


class Outs:
    """host and device output buffers of one call"""

    def __init__(self, nq, k=K):
        import torch
        self.h = (np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64), np.zeros(nq, np.uint32))
        self.d = (torch.zeros((nq, k), dtype=torch.int64, device="cuda"),
                  torch.zeros((nq, k), dtype=torch.float64, device="cuda"),
                  torch.zeros(nq, dtype=torch.int32, device="cuda"))

    def hp(self):
        return tuple(a.ctypes.data for a in self.h)

    def dp(self):
        return tuple(a.data_ptr() for a in self.d)

    def host(self):
        return tuple(a.tobytes() for a in self.h)

    def device(self):
        import torch
        torch.cuda.synchronize()
        return tuple(a.cpu().numpy().tobytes() for a in self.d)


def make_col(ctx, b):
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, DIM, "COSINE", "F32", capacity=N)
    col.append(b.corpus)
    col.finalize()
    return col


def submit(L, col, b, kind, filtered, o, nq=None, cancel=None):
    """hand the batch to entry point `kind`: (status, ticket or None, True for a sharded ticket)"""
    h, nq = col.h, b.nq if nq is None else nq
    t = C.c_uint32()
    fh = (b.f.ctypes.data, 2, b.qf.ctypes.data)
    fd = (b.df.data_ptr(), 2, b.qf.ctypes.data)
    q, dq = b.q.ctypes.data, b.dq.data_ptr()
    if kind == "blocking_host":
        st = (L.sdb_knn_bruteforce_filtered(h, q, nq, K, *fh, *o.hp(), cancel) if filtered
              else L.sdb_knn_bruteforce(h, q, nq, K, *o.hp(), cancel))
        return st, None, False
    if kind == "blocking_device":
        st = (L.sdb_knn_bruteforce_filtered_device(h, dq, nq, K, *fd, 0, *o.dp()) if filtered
              else L.sdb_knn_bruteforce_device(h, dq, nq, K, 0, *o.dp()))
        return st, None, False
    if kind == "ticket_host":
        st = (L.sdb_knn_submit_filtered(h, q, nq, K, *fh, *o.hp(), C.byref(t)) if filtered
              else L.sdb_knn_submit(h, q, nq, K, *o.hp(), C.byref(t)))
        return st, t.value, False
    if kind == "ticket_device":
        st = (L.sdb_knn_submit_filtered_device(h, dq, nq, K, *fd, 0, *o.dp(), C.byref(t)) if filtered
              else L.sdb_knn_submit_device(h, dq, nq, K, 0, *o.dp(), C.byref(t)))
        return st, t.value, False
    if kind == "sharded_host":
        st = (L.sdb_knn_sharded_submit_filtered(h, q, nq, K, *fh, N, *o.hp(), C.byref(t)) if filtered
              else L.sdb_knn_sharded_submit(h, q, nq, K, *o.hp(), C.byref(t)))
        return st, t.value, True
    if kind == "sharded_device":
        st = (L.sdb_knn_sharded_submit_filtered_device(h, dq, nq, K, *fd, N, *o.dp(), C.byref(t)) if filtered
              else L.sdb_knn_sharded_submit_device(h, dq, nq, K, *o.dp(), C.byref(t)))
        return st, t.value, True
    assert kind == "sharded_multi"
    hs = (C.c_void_p * 1)(h)
    st = (L.sdb_knn_sharded_multi_filtered(hs, 1, q, nq, K, *fh, N, *o.hp()) if filtered
          else L.sdb_knn_sharded_multi(hs, 1, q, nq, K, *o.hp()))
    return st, None, False


def wait(L, col, ticket, sharded):
    return L.sdb_knn_sharded_wait(col.h, ticket) if sharded else L.sdb_knn_wait(col.h, ticket)


def result(kind, o):
    return o.device() if kind.endswith("_device") else o.host()


ALL = UNSHARDED + SHARDED


@pytest.mark.parametrize("filtered", [False, True], ids=["unfiltered", "filtered"])
def test_every_variant_gives_the_same_bytes(filtered):
    from surrealdb_b200 import Context
    from surrealdb_b200 import _lib
    L = _lib.lib()
    live0 = live()
    ctx = Context(0)
    b = Batch()
    col = make_col(ctx, b)
    o = Outs(b.nq)
    st, t, sh = submit(L, col, b, "blocking_host", filtered, o)  # settles the corpus' remembered rung
    assert st == 0
    want = o.host()
    launches = {}
    for kind in ALL:
        o = Outs(b.nq)
        st, t, sh = submit(L, col, b, kind, filtered, o)
        assert st == 0, (kind, L.sdb_last_error())
        if t is not None:
            assert wait(L, col, t, sh) == 0, (kind, L.sdb_last_error())
        assert result(kind, o) == want, kind
        launches[kind] = launches_of(col)
    print(filtered, launches)
    assert len({launches[kd] for kd in UNSHARDED}) == 1, launches
    assert len({launches[kd] for kd in SHARDED}) == 1, launches
    assert int(np.frombuffer(want[2], np.uint32).min()) == K
    col.close()
    ctx.close()
    assert live() == live0


def test_row_base_of_each_entry_point():
    # host-buffer calls and sharded calls rank with the corpus' row_base, device-buffer calls with their argument
    from surrealdb_b200 import Context
    from surrealdb_b200 import _lib
    L = _lib.lib()
    live0 = live()
    ctx = Context(0)
    b = Batch(nq=8, seed=6)
    col = make_col(ctx, b)
    o = Outs(b.nq)
    assert submit(L, col, b, "blocking_host", False, o)[0] == 0
    base_rows = o.h[0].copy()
    col.set_row_base(77)
    t = C.c_uint32()
    for kind in ALL:
        o = Outs(b.nq)
        if kind == "blocking_device":
            assert L.sdb_knn_bruteforce_device(col.h, b.dq.data_ptr(), b.nq, K, 5, *o.dp()) == 0
        elif kind == "ticket_device":
            assert L.sdb_knn_submit_device(col.h, b.dq.data_ptr(), b.nq, K, 5, *o.dp(), C.byref(t)) == 0
            assert L.sdb_knn_wait(col.h, t.value) == 0
        else:
            st, tk, sh = submit(L, col, b, kind, False, o)
            assert st == 0
            if tk is not None:
                assert wait(L, col, tk, sh) == 0
        shift = 5 if kind in ("blocking_device", "ticket_device") else 77
        rows = np.frombuffer(result(kind, o)[0], np.uint64).reshape(b.nq, K)
        assert (rows == base_rows + np.uint64(shift)).all(), kind
    col.close()
    ctx.close()
    assert live() == live0


def test_empty_batches_cancel_flags_full_tickets_and_stale_waits():
    from surrealdb_b200 import Context
    from surrealdb_b200 import _lib
    L = _lib.lib()
    live0 = live()
    ctx = Context(0)
    b = Batch(nq=16, seed=7)
    col = make_col(ctx, b)
    o = Outs(b.nq)
    assert submit(L, col, b, "blocking_host", False, o)[0] == 0
    want = {False: o.host()}
    assert submit(L, col, b, "blocking_host", True, o)[0] == 0
    want[True] = o.host()

    # ---- nq == 0 ----
    t = C.c_uint32()
    stats0 = col.stats()
    l0 = L.sdb_ctx_kernel_launches(ctx.h)
    assert L.sdb_knn_bruteforce(col.h, None, 0, K, None, None, None, None) == 0
    assert L.sdb_knn_bruteforce_device(col.h, None, 0, K, 0, None, None, None) == 0
    for filtered in (False, True):
        for kind in ("blocking_host", "blocking_device"):
            assert submit(L, col, b, kind, filtered, o, nq=0)[0] == 0, (kind, filtered)
    one = np.ones(1, np.int32)
    assert submit(L, col, b, "blocking_host", False, o, nq=0, cancel=one.ctypes.data)[0] == 0
    assert submit(L, col, b, "blocking_host", True, o, nq=0, cancel=one.ctypes.data)[0] == 0
    assert L.sdb_ctx_kernel_launches(ctx.h) == l0 and col.stats() == stats0  # no work at all
    for filtered in (False, True):
        assert submit(L, col, b, "ticket_host", filtered, o, nq=0)[0] == _lib.SDB_EINVAL
        for kind in ("sharded_host", "sharded_device", "sharded_multi"):
            assert submit(L, col, b, kind, filtered, o, nq=0)[0] == _lib.SDB_EINVAL, (kind, filtered)
    st, tk, _ = submit(L, col, b, "ticket_device", False, o, nq=0)
    assert st == 0
    assert L.sdb_ctx_kernel_launches(ctx.h) == l0  # a ticket, no kernels
    assert L.sdb_knn_wait(col.h, tk) == 0
    st, tk, _ = submit(L, col, b, "ticket_device", True, o, nq=0)
    assert st == 0 and L.sdb_knn_wait(col.h, tk) == 0

    # ---- cancel: the per-call flag of the blocking host calls, the context's flag everywhere ----
    assert submit(L, col, b, "blocking_host", False, o, cancel=one.ctypes.data)[0] == _lib.SDB_ECANCELLED
    assert submit(L, col, b, "blocking_host", True, o, cancel=one.ctypes.data)[0] == _lib.SDB_ECANCELLED
    L.sdb_ctx_cancel(ctx.h)
    for filtered in (False, True):
        for kind in ALL:
            assert submit(L, col, b, kind, filtered, o)[0] == _lib.SDB_ECANCELLED, (kind, filtered)
    L.sdb_ctx_cancel_reset(ctx.h)

    # ---- four tickets in flight: every entry point refuses a fifth batch ----
    kinds = (("ticket_host", False), ("ticket_device", True), ("sharded_host", True), ("sharded_device", False))
    flight = []
    for kind, filtered in kinds:
        ob = Outs(b.nq)
        st, tk, sh = submit(L, col, b, kind, filtered, ob)
        assert st == 0, (kind, L.sdb_last_error())
        flight.append((kind, filtered, ob, tk, sh))
    for filtered in (False, True):
        for kind in ALL:
            assert submit(L, col, b, kind, filtered, o)[0] == _lib.SDB_EOVERFLOW, (kind, filtered)
    assert L.sdb_debug_screen_batch(col.h, b.q.ctypes.data, b.nq, K, 2, 1, 4096, 0, *([None] * 8)) == _lib.SDB_EOVERFLOW
    for kind, filtered, ob, tk, sh in reversed(flight):
        assert wait(L, col, tk, sh) == 0, (kind, L.sdb_last_error())
        assert result(kind, ob) == want[filtered], kind

    # ---- stale and unknown tickets ----
    for kind, filtered, ob, tk, sh in flight:
        assert wait(L, col, tk, sh) == _lib.SDB_EINVAL, kind
    assert L.sdb_knn_wait(col.h, 123456) == _lib.SDB_EINVAL
    assert L.sdb_knn_sharded_wait(col.h, 123456) == _lib.SDB_EINVAL

    # ---- the column still answers, and four tickets fit again ----
    for kind in ALL:
        o = Outs(b.nq)
        st, tk, sh = submit(L, col, b, kind, True, o)
        assert st == 0
        if tk is not None:
            assert wait(L, col, tk, sh) == 0
        assert result(kind, o) == want[True], kind
    col.close()
    ctx.close()
    assert live() == live0

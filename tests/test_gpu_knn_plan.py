"""A brute-force batch in flight keeps the plan it was submitted with.  The corpus' screen and exact settings at submit
decide how its wait climbs the ladder, repairs it and remembers the rung it settled on; setters called between the
submit and the wait apply to later batches only.

The column holds DUP copies of one vector among random rows, and every query lies close to it: each query's candidate
set holds every copy, which overflows the 4096-entry lists of the first rung, so the whole batch climbs at its wait."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, DIM, NQ, K, DUP = 20_000, 128, 64, 10, 6000


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def data():
    rng = np.random.default_rng(11)
    corpus = rng.standard_normal((N, DIM)).astype(np.float32)
    v = corpus[0].copy()
    corpus[rng.choice(N, DUP, replace=False)] = v
    queries = np.ascontiguousarray(v + 1e-3 * rng.standard_normal((NQ, DIM)), np.float64)
    return corpus, queries


def make_col(ctx, corpus):
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, DIM, "COSINE", "F32", capacity=N)
    col.append(corpus)
    col.finalize()
    return col


def run(col, queries, between=None):
    """one ticket of the batch; between() runs after its submit and before its wait -> (rows, dist, count, stats)"""
    rows, dist, cnt = np.zeros((NQ, K), np.uint64), np.zeros((NQ, K), np.float64), np.zeros(NQ, np.uint32)
    t = col.submit_host(queries.ctypes.data, NQ, K, rows.ctypes.data, dist.ctypes.data, cnt.ctypes.data)
    if between:
        between()
    col.wait(t)
    stats = col.stats()
    del stats["screen_ms"], stats["total_ms"]
    return rows, dist, cnt, stats


def same(a, b):
    ra, da, ca, sa = a
    rb, db, cb, sb = b
    assert np.array_equal(ca, cb) and np.array_equal(ra, rb)
    assert da.tobytes() == db.tobytes()
    assert sa == sb


def test_setters_between_submit_and_wait_do_not_change_the_batch(ctx):
    corpus, queries = data()
    ref_col, col = make_col(ctx, corpus), make_col(ctx, corpus)
    first, again = run(ref_col, queries), run(ref_col, queries)
    assert (first[2] == K).all()
    # the first batch climbed at its wait; the second started on the rung the first one settled on
    assert first[3]["kernel_launches"] > again[3]["kernel_launches"]
    assert first[3]["screen_used"] == again[3]["screen_used"]

    def change_settings():
        col.set_exact(False)
        col.set_screen("NONE_EXACT")

    same(run(col, queries, change_settings), first)
    col.set_screen("AUTO")
    col.set_exact(True)
    same(run(col, queries), again)  # remembered under the key of the plan the batch was submitted with

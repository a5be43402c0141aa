"""The int8 tensor-core screen's streaming pass hands its survivors to a drain warp through a small ring in shared
memory.  These cases fill that ring many times within one work item (a crowd of identical rows that half the queries
of every 128-query block keep) and launch an even and an odd number of query blocks; the results must be the exact
kernel's, bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def _col(ctx, corpus, screen):
    from surrealdb_b200 import VectorColumn
    col = VectorColumn(ctx, corpus.shape[1], "COSINE", "F32", capacity=corpus.shape[0])
    col.append(corpus)
    col.finalize()
    col.set_screen(screen)
    return col


@pytest.mark.parametrize("nq", [256, 384])  # 2 and 3 query blocks of 128
@pytest.mark.parametrize("k", [10, 100])
def test_int8_streaming_crowd_matches_exact(ctx, nq, k):
    rng = np.random.default_rng(nq + k)
    n, dim = 40000, 128
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    corpus[5000:5600] = corpus[5000]  # 600 identical rows: every tile they fill has 256 survivors per crowd query
    queries = rng.uniform(-1, 1, (nq, dim))
    queries[::2] = corpus[5000] + rng.normal(0, 1e-3, (nq // 2, dim))
    col = _col(ctx, corpus, "TC_INT8")
    rows, dist, cnt = col.knn(queries, k)
    st = col.stats()
    assert st["screen_used"] == 4 and st["n_passes"] == 2, st  # probe + streaming pass
    want_rows, want_dist, want_cnt = _col(ctx, corpus, "NONE_EXACT").knn(queries, k)
    assert (cnt == k).all() and np.array_equal(cnt, want_cnt)
    assert rows.tobytes() == want_rows.tobytes()
    assert dist.tobytes() == want_dist.tobytes()

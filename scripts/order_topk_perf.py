#!/usr/bin/env python
"""Queries/s of `ORDER BY vector::<fn>(emb, $q) ASC|DESC LIMIT k` (sdb_corpus_order_topk) on one cached column:

  * vector::similarity::cosine DESC on a COSINE column (the screens + the similarity proof) against sdb_knn_bruteforce
    on the same column and batch;
  * vector::similarity::pearson DESC on a PEARSON column (the exact kernel) against the exact kernel's KNN ranking
    (sdb_knn_bruteforce with NONE_EXACT) on the same column;
  * vector::dot DESC (maximum inner product, the bf16 screen + the dot proof) on the COSINE column and on a EUCLIDEAN
    one, each against sdb_knn_bruteforce on the same column and against the exact kernel (NONE_EXACT, --exact-max
    queries), with the survivors per query and the repaired / fallback counts;
  * the cross views, each against the same column's KNN and the exact kernel like the dot rows: cosine distance DESC
    and euclidean DESC (farthest first) on the COSINE column, similarity DESC and euclidean DESC on the EUCLIDEAN one;
  * the route without this call: sdb_corpus_project per query (every row's value copied to the host) and a host top-k
    (numpy argpartition + sort), timed on --project-max queries and scaled.

  python scripts/order_topk_perf.py [--n 10000000 --dim 768 --k 10 --batch 1024 --reps 3 --exact-max 4
                                     --project-max 4 --pearson-n 10000000 --dot-euclid-n 10000000
                                     --out order_topk_perf.json]

The rows are the library's synthetic rows (append_synthetic), the queries gen_f32 values of another seed.  Each rate
is the batch over the median of --reps synchronous calls after one warm-up call.  10 queries of the batch are checked
bit for bit against NONE_EXACT (the exact kernel).  The card's name and power limit are read in the same call.  Prints
one JSON line per row and a summary line; writes them to --out as well.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:  # the timing itself does not depend on it
        return f"unknown ({e})"


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()  # synchronous: returns once the results are on the host
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), [min(ts) * 1e3, max(ts) * 1e3]


def host_topk(col, Q, k, fn):
    """the route without sdb_corpus_order_topk: every row's value to the host, then a host top-k (DESC)"""
    for q in Q:
        v = col.project(fn, q)
        part = np.argpartition(-v, k)[:k]
        part[np.argsort(-v[part], kind="stable")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--exact-max", type=int, default=4)
    ap.add_argument("--project-max", type=int, default=4)
    ap.add_argument("--pearson-n", type=int, default=10_000_000)
    ap.add_argument("--dot-euclid-n", type=int, default=10_000_000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from surrealdb_b200 import Context, VectorColumn
    from surrealdb_b200.synthetic import gen_f32

    if not torch.cuda.is_available():
        raise SystemExit("order_topk_perf.py needs a CUDA device")
    ctx = Context(0)
    B, k = a.batch, a.k
    Q = gen_f32(0x5DB1, 0, B * a.dim).reshape(B, a.dim).astype(np.float64)
    lines = []

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        lines.append(line)

    summary = {"config": f"{a.n}x{a.dim} F32 synthetic", "k": k, "batch": B, "gpu": gpu_info()}

    def dot_rows(col, column, t_knn, fn="DOT", order="DESC"):
        """fn / order (vector::dot DESC by default) on col: the screened batch, the exact kernel on a few queries,
        parity on 10"""
        t_dot, sp_dot = timed(lambda: col.order_topk(Q, k, fn, order), a.reps)
        st = col.stats()
        Be = min(B, a.exact_max)
        col.set_screen("NONE_EXACT")
        t_ex, sp_ex = timed(lambda: col.order_topk(Q[:Be], k, fn, order), a.reps)
        ref = col.order_topk(Q[:10], k, fn, order)
        col.set_screen("AUTO")
        got = col.order_topk(Q[:10], k, fn, order)
        summary[f"{fn.lower()}_{order.lower()}_{column.lower()}_parity_10_vs_exact"] = all(
            u.tobytes() == v.tobytes() for u, v in zip(got, ref))
        emit({"fn": fn, "order": order, "column": column, "batch": B, "order_qps": B / t_dot,
              "knn_qps": B / t_knn, "order_over_knn_time": t_dot / t_knn, "order_spread_ms": sp_dot,
              "exact_timed_queries": Be, "exact_qps": Be / t_ex, "exact_spread_ms": sp_ex,
              "screen_used": st["screen_used"], "screen_ms": st["screen_ms"], "total_ms": st["total_ms"],
              "survivors_per_query": st["n_survivors"] / B, "largest_candidate_set": st["n_candidates"],
              "n_fallback": st["n_fallback"], "n_repaired": st["n_repaired"]})

    col = VectorColumn(ctx, a.dim, "COSINE", "F32", capacity=a.n)
    col.append_synthetic(seed=0x5DB0, first_row=0, n=a.n)
    col.finalize()
    t_knn, sp_knn = timed(lambda: col.knn(Q, k), a.reps)
    st_knn = col.stats()
    t_ord, sp_ord = timed(lambda: col.order_topk(Q, k, "SIMILARITY_COSINE", "DESC"), a.reps)
    st = col.stats()
    emit({"fn": "SIMILARITY_COSINE", "order": "DESC", "column": "COSINE", "batch": B, "order_qps": B / t_ord,
          "knn_qps": B / t_knn, "order_over_knn_time": t_ord / t_knn, "order_spread_ms": sp_ord,
          "knn_spread_ms": sp_knn, "screen_used": st["screen_used"], "screen_ms": st["screen_ms"],
          "total_ms": st["total_ms"], "n_fallback": st["n_fallback"], "n_repaired": st["n_repaired"],
          "knn_screen_used": st_knn["screen_used"], "knn_n_fallback": st_knn["n_fallback"]})
    Pm = min(B, a.project_max)
    t_proj, sp_proj = timed(lambda: host_topk(col, Q[:Pm], k, "SIMILARITY_COSINE"), a.reps)
    emit({"fn": "SIMILARITY_COSINE", "order": "DESC", "route": "project + host top-k", "timed_queries": Pm,
          "qps": Pm / t_proj, "spread_ms": sp_proj, "order_speedup_per_query": (t_proj / Pm) / (t_ord / B)})
    Qp = Q[:10]
    got = col.order_topk(Qp, k, "SIMILARITY_COSINE", "DESC")
    col.set_screen("NONE_EXACT")
    ref = col.order_topk(Qp, k, "SIMILARITY_COSINE", "DESC")
    col.set_screen("AUTO")
    summary["cosine_desc_parity_10_vs_exact"] = all(u.tobytes() == v.tobytes() for u, v in zip(got, ref))
    dot_rows(col, "COSINE", t_knn)
    dot_rows(col, "COSINE", t_knn, "COSINE", "DESC")
    dot_rows(col, "COSINE", t_knn, "EUCLIDEAN", "DESC")
    col.close()
    del col
    torch.cuda.empty_cache()

    if a.dot_euclid_n:
        col = VectorColumn(ctx, a.dim, "EUCLIDEAN", "F32", capacity=a.dot_euclid_n)
        col.append_synthetic(seed=0x5DB0, first_row=0, n=a.dot_euclid_n)
        col.finalize()
        t_knn, _ = timed(lambda: col.knn(Q, k), a.reps)
        dot_rows(col, "EUCLIDEAN", t_knn)
        dot_rows(col, "EUCLIDEAN", t_knn, "SIMILARITY_COSINE", "DESC")
        dot_rows(col, "EUCLIDEAN", t_knn, "EUCLIDEAN", "DESC")
        col.close()
    del col
    torch.cuda.empty_cache()

    if a.pearson_n:
        col = VectorColumn(ctx, a.dim, "PEARSON", "F32", capacity=a.pearson_n)
        col.append_synthetic(seed=0x5DB0, first_row=0, n=a.pearson_n)
        col.finalize()
        Be = min(B, a.exact_max)
        t_ord, sp_ord = timed(lambda: col.order_topk(Q[:Be], k, "PEARSON", "DESC"), a.reps)
        col.set_screen("NONE_EXACT")
        t_ex, sp_ex = timed(lambda: col.knn(Q[:Be], k), a.reps)
        col.set_screen("AUTO")
        emit({"fn": "PEARSON", "order": "DESC", "column": "PEARSON", "rows": a.pearson_n, "timed_queries": Be,
              "order_qps": Be / t_ord, "exact_knn_qps": Be / t_ex, "order_spread_ms": sp_ord,
              "exact_spread_ms": sp_ex})
        col.close()
    emit(summary)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

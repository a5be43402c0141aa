#!/usr/bin/env python
"""Queries/s of brute-force PEARSON KNN through the cosine tensor-core screens on the centred rows (AUTO) against the
exact kernel (NONE_EXACT) on one column, and the screen time of a COSINE column of the same rows beside it.

  python scripts/pearson_knn_perf.py [--n 10000000 --dim 768 --k 10 --batches 1,8,64,1024 --reps 3
                                      --f64-n 5000000 --out pearson_knn_perf.json]

The F32 rows are the library's synthetic rows (append_synthetic), the queries gen_f32 values of another seed.  For each
batch size the two screens alternate in one loop (one warm-up call each first); each rate is the batch over the median
of --reps synchronous calls.  The exact kernel makes two passes over the corpus per query, so batches above
--exact-max are timed at --exact-max queries and scaled (marked "scaled").  Also reported per AUTO row: the library's
screen time, fallback / repair counts and the largest candidate set.  Then: a COSINE column of the same rows at the
largest batch (screen time of the same kernel on the same bytes), two filtered batches of 64 (a filter passing 1 % of
the rows, and one passing 4000 rows: the direct regime), and an F64 column of --f64-n rows (the same synthetic values
stored as f64) at the largest batch.  10 queries of the last batch are checked bit for bit against NONE_EXACT on each
PEARSON column.  The card's name and power limit are read in the same call.  Prints one JSON line per row and a
summary line; writes them to --out as well.
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


def call(col, Q, k, **kw):
    t0 = time.perf_counter()
    r = col.knn(Q, k, **kw)  # synchronous: returns once the results are on the host
    return time.perf_counter() - t0, r, col.stats()


def parity(col, Qp, k):
    col.set_screen("AUTO")
    _, (r_a, d_a, c_a), _ = call(col, Qp, k)
    col.set_screen("NONE_EXACT")
    _, (r_e, d_e, c_e), _ = call(col, Qp, k)
    col.set_screen("AUTO")
    return bool(np.array_equal(r_a, r_e) and d_a.tobytes() == d_e.tobytes() and np.array_equal(c_a, c_e))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--batches", default="1,8,64,1024")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--exact-max", type=int, default=8)
    ap.add_argument("--f64-n", type=int, default=5_000_000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from surrealdb_b200 import Context, VectorColumn
    from surrealdb_b200.engine import pack_row_filter
    from surrealdb_b200.synthetic import gen_f32

    if not torch.cuda.is_available():
        raise SystemExit("pearson_knn_perf.py needs a CUDA device")
    ctx = Context(0)
    batches = [int(b) for b in a.batches.split(",")]
    Bmax = max(batches)
    Qall = gen_f32(0x5DB1, 0, Bmax * a.dim).reshape(Bmax, a.dim).astype(np.float64)
    Qp = Qall[Bmax - 10:Bmax]
    lines = []

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        lines.append(line)

    summary = {"config": f"{a.n}x{a.dim} F32 synthetic", "k": a.k, "gpu": gpu_info()}

    def timed(col, Q, **kw):
        call(col, Q, a.k, **kw)
        ts, st = [], None
        for _ in range(a.reps):
            t, _, st = call(col, Q, a.k, **kw)
            ts.append(t)
        return float(np.median(ts)), st

    col = VectorColumn(ctx, a.dim, "PEARSON", "F32", capacity=a.n)
    col.append_synthetic(seed=0x5DB0, first_row=0, n=a.n)
    col.finalize()
    for B in batches:
        Q = Qall[:B]
        Be = min(B, a.exact_max)
        col.set_screen("AUTO")
        call(col, Q, a.k)
        col.set_screen("NONE_EXACT")
        call(col, Q[:Be], a.k)
        ta, te, st = [], [], None
        for _ in range(a.reps):
            col.set_screen("AUTO")
            t, _, st = call(col, Q, a.k)
            ta.append(t)
            col.set_screen("NONE_EXACT")
            te.append(call(col, Q[:Be], a.k)[0] * B / Be)
        t_a, t_e = float(np.median(ta)), float(np.median(te))
        emit({"metric": "PEARSON", "dtype": "F32", "batch": B, "auto_qps": B / t_a, "exact_qps": B / t_e,
              "speedup": t_e / t_a, "exact_timed_queries": Be, "exact_scaled": Be != B,
              "auto_spread_ms": [min(ta) * 1e3, max(ta) * 1e3], "exact_spread_ms": [min(te) * 1e3, max(te) * 1e3],
              "screen_used": st["screen_used"], "screen_ms": st["screen_ms"], "total_ms": st["total_ms"],
              "n_fallback": st["n_fallback"], "n_repaired": st["n_repaired"], "max_candidates": st["n_candidates"]})
    rng = np.random.default_rng(3)
    col.set_screen("AUTO")
    for label, mask in (("filter_1pct", rng.random(a.n) < 0.01), ("filter_4000_rows", np.zeros(a.n, bool))):
        if label == "filter_4000_rows":
            mask[rng.choice(a.n, 4000, replace=False)] = True
        t, st = timed(col, Qall[:64], filters=pack_row_filter(mask))
        emit({"metric": "PEARSON", "dtype": "F32", "batch": 64, "filter": label, "auto_qps": 64 / t,
              "n_passes": st["n_passes"], "screen_ms": st["screen_ms"], "n_fallback": st["n_fallback"]})
    summary["PEARSON_F32_parity_10_vs_exact"] = parity(col, Qp, a.k)
    col.close()
    del col
    torch.cuda.empty_cache()

    col = VectorColumn(ctx, a.dim, "COSINE", "F32", capacity=a.n)  # the same kernel on the same bytes
    col.append_synthetic(seed=0x5DB0, first_row=0, n=a.n)
    col.finalize()
    t, st = timed(col, Qall)
    emit({"metric": "COSINE", "dtype": "F32", "batch": Bmax, "auto_qps": Bmax / t, "screen_used": st["screen_used"],
          "screen_ms": st["screen_ms"], "total_ms": st["total_ms"], "n_fallback": st["n_fallback"]})
    col.close()
    del col
    torch.cuda.empty_cache()

    if a.f64_n:
        col = VectorColumn(ctx, a.dim, "PEARSON", "F64", capacity=a.f64_n)
        chunk = 250_000
        for r0 in range(0, a.f64_n, chunk):
            m = min(chunk, a.f64_n - r0)
            col.append(gen_f32(0x5DB0, r0 * a.dim, m * a.dim).reshape(m, a.dim).astype(np.float64))
        col.finalize()
        Be = min(Bmax, a.exact_max)
        col.set_screen("NONE_EXACT")
        te, _ = timed(col, Qall[:Be])
        col.set_screen("AUTO")
        t, st = timed(col, Qall)
        emit({"metric": "PEARSON", "dtype": "F64", "rows": a.f64_n, "batch": Bmax, "auto_qps": Bmax / t,
              "exact_qps": Be / te, "exact_timed_queries": Be, "speedup": (te * Bmax / Be) / t,
              "screen_used": st["screen_used"], "screen_ms": st["screen_ms"], "total_ms": st["total_ms"],
              "n_fallback": st["n_fallback"], "n_repaired": st["n_repaired"], "max_candidates": st["n_candidates"]})
        summary["PEARSON_F64_parity_10_vs_exact"] = parity(col, Qp, a.k)
        col.close()
    emit(summary)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Filtered brute-force KNN (sdb_knn_bruteforce_filtered) on a large cached column, against the two ways a residual
WHERE was served before: the unfiltered call, and set_skip(~filter) + finalize followed by the unfiltered call.

  python scripts/filtered_knn_perf.py [--n 10000000 --dim 768 --nq 1024 --k 10 --reps 3 --out filtered_knn_perf.json]

The column is append_synthetic rows (F32, cosine).  Queries are corpus rows plus a little noise.  Filters: random
row filters at 100 / 50 / 10 / 1 / 0.1 / 0.05 / 0.04 / 0.01 % density (the last two
pass at most 4096 rows of 10M: the direct regime) and a contiguous 10 % row range, each shared by the whole batch,
and 64 distinct random 10 % filters spread over the batch.  For every filter: queries/s of a batch of nq and of a batch
of 1 (median of --reps synchronous calls after one warm-up), and the library's screen_ms, n_fallback, n_repaired and
n_candidates of the last batch.  In the same run, alternated --reps times: the unfiltered call, and set_skip + finalize
with a 10 % filter (the cost a statement paid before the filtered call existed).  The GPU's name and power limit are
printed with the numbers.  Prints one JSON line; writes it to --out as well.
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
    fn()  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    from surrealdb_b200 import Context, VectorColumn, pack_row_filter

    ctx = Context(0)
    res = {"config": f"{a.n}x{a.dim} F32 cosine append_synthetic", "nq": a.nq, "k": a.k, "gpu": gpu_info()}
    col = VectorColumn(ctx, a.dim, "COSINE", "F32", capacity=a.n)
    for r0 in range(0, a.n, 1 << 20):
        col.append_synthetic(11, r0, min(1 << 20, a.n - r0))
    t0 = time.perf_counter()
    col.finalize()
    res["finalize_ms"] = (time.perf_counter() - t0) * 1e3
    rng = np.random.default_rng(3)
    idx = rng.choice(a.n, a.nq, replace=False)
    Q = np.stack([col.read_rows(int(i), 1)[0] for i in idx]).astype(np.float64)
    Q += rng.normal(0, 0.05 * float(np.abs(Q).mean()), Q.shape)

    def stats_of(prefix, st):
        for key in ("screen_ms", "n_fallback", "n_repaired", "n_candidates"):
            res[f"{prefix}_{key}"] = st[key]

    t = timed(lambda: col.knn(Q, a.k), a.reps)
    res["unfiltered_qps"] = a.nq / t
    stats_of("unfiltered", col.stats())
    res["unfiltered_1q_ms"] = timed(lambda: col.knn(Q[:1], a.k), a.reps) * 1e3

    filters = {f"random_{p * 100:g}pct": rng.random(a.n) < p for p in (1.0, 0.5, 0.1, 0.01, 0.001, 0.0005, 0.0004, 0.0001)}
    rng_mask = np.zeros(a.n, bool)
    rng_mask[a.n // 3 : a.n // 3 + a.n // 10] = True
    filters["range_10pct"] = rng_mask
    for name, m in filters.items():
        f = pack_row_filter(m)
        t = timed(lambda: col.knn(Q, a.k, filters=f), a.reps)
        res[f"{name}_qps"] = a.nq / t
        stats_of(name, col.stats())
        res[f"{name}_1q_ms"] = timed(lambda: col.knn(Q[:1], a.k, filters=f), a.reps) * 1e3

    f64 = pack_row_filter(rng.random((64, a.n)) < 0.1)
    qf = (np.arange(a.nq) % 64).astype(np.uint32)
    t = timed(lambda: col.knn(Q, a.k, filters=f64, query_filter=qf), a.reps)
    res["distinct64_10pct_qps"] = a.nq / t
    stats_of("distinct64_10pct", col.stats())

    # before the filtered call: the statement's predicate went into the skip mask and the column was re-finalized
    m10 = filters["random_10pct"]
    unf, skip_fin, filt = [], [], []
    f10 = pack_row_filter(m10)
    for _ in range(a.reps):
        t0 = time.perf_counter()
        col.knn(Q, a.k)
        unf.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        col.set_skip((~m10).astype(np.uint8))
        col.finalize()
        skip_fin.append(time.perf_counter() - t0)
        col.knn(Q, a.k)
        col.set_skip(None)
        col.finalize()
        t0 = time.perf_counter()
        col.knn(Q, a.k, filters=f10)
        filt.append(time.perf_counter() - t0)
    res["alt_unfiltered_ms"] = float(np.median(unf)) * 1e3
    res["alt_set_skip_finalize_ms"] = float(np.median(skip_fin)) * 1e3
    res["alt_filtered_10pct_ms"] = float(np.median(filt)) * 1e3
    col.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

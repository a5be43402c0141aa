#!/usr/bin/env python
"""Queries/s of brute-force cosine KNN on an F64 column (screened on the tensor cores) against the same data stored
as F32, and the exact kernel's per-query time on the F64 column.

  python scripts/f64_knn_perf.py [--n 5000000 --dim 768 --nq 1024 --k 10 --reps 5 --out f64_knn_perf.json]

The rows are uniform(-20, 20) f64 drawn on the device chunk by chunk (not f32 values); the F32 column holds their f32
roundings.  The two columns are built one after the other, so that only one is resident at a time (5M x 768: 42 GB
for the F64 rows and their bf16 / int8 copies).  Each rate is nq over the median of --reps synchronous calls after
one warm-up call.  Also reported: the library's screen time, fallback / repair counts and the largest candidate set
of the last AUTO call, the exact kernel (SDB_SCREEN_NONE_EXACT) on 8 queries, and whether 10 AUTO answers equal the
exact kernel's bit for bit.  Prints one JSON line; writes it to --out as well.
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


def fill(col, torch, n, dim, dtype, seed, chunk=65536):
    g = torch.Generator(device="cuda").manual_seed(seed)
    for r0 in range(0, n, chunk):
        m = min(chunk, n - r0)
        x = torch.rand((m, dim), dtype=torch.float64, device="cuda", generator=g) * 40.0 - 20.0
        if dtype == "F32":
            x = x.to(torch.float32)
        torch.cuda.synchronize()
        col.append_device(x.data_ptr(), m)
        del x
    torch.cuda.empty_cache()
    col.finalize()


def timed(col, Q, k, reps):
    col.knn(Q, k)  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        col.knn(Q, k)  # synchronous: returns once the results are on the host
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), col.stats()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=5_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from surrealdb_b200 import Context, VectorColumn

    if not torch.cuda.is_available():
        raise SystemExit("f64_knn_perf.py needs a CUDA device")
    ctx = Context(0)
    rng = np.random.default_rng(1)
    Q = rng.uniform(-20, 20, (a.nq, a.dim))
    res = {"config": f"{a.n}x{a.dim} cosine uniform(-20,20)", "nq": a.nq, "k": a.k, "gpu": gpu_info()}

    col = VectorColumn(ctx, a.dim, "COSINE", "F64", capacity=a.n)
    fill(col, torch, a.n, a.dim, "F64", 7)
    t, st = timed(col, Q, a.k, a.reps)
    res["f64_auto_qps"] = a.nq / t
    res["f64_auto_screen"] = st["screen_used"]
    res["lib_screen_ms"] = st["screen_ms"]
    res["lib_total_ms"] = st["total_ms"]
    for key in ("n_fallback", "n_repaired", "n_candidates", "n_special_rows"):
        res[key] = st[key]
    r_auto, d_auto, _ = col.knn(Q[:10], a.k)
    col.set_screen("NONE_EXACT")
    col.knn(Q[:1], a.k)  # warm-up
    t0 = time.perf_counter()
    col.knn(Q[:8], a.k)
    res["exact_ms_per_query"] = (time.perf_counter() - t0) / 8 * 1e3
    res["exact_qps"] = 1e3 / res["exact_ms_per_query"]
    r_ex, d_ex, _ = col.knn(Q[:10], a.k)
    res["parity_10_vs_exact"] = bool(np.array_equal(r_auto, r_ex) and d_auto.tobytes() == d_ex.tobytes())
    col.close()
    del col
    torch.cuda.empty_cache()

    col = VectorColumn(ctx, a.dim, "COSINE", "F32", capacity=a.n)
    fill(col, torch, a.n, a.dim, "F32", 7)
    t, st = timed(col, Q, a.k, a.reps)
    res["f32_auto_qps"] = a.nq / t
    res["f32_auto_screen"] = st["screen_used"]
    res["f32_lib_screen_ms"] = st["screen_ms"]
    col.close()

    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

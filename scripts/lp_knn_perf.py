#!/usr/bin/env python
"""Queries/s of brute-force MANHATTAN, CHEBYSHEV and MINKOWSKI KNN through the f32 screen (AUTO) against the exact
kernel (NONE_EXACT) on one column.

  python scripts/lp_knn_perf.py [--n 10000000 --dim 768 --k 10 --batches 1,8,32,64,1024 --reps 3 --out lp_knn_perf.json]
  python scripts/lp_knn_perf.py --metrics MINKOWSKI --orders 2,3,4,8 [--dtype F64 --n 5000000 --batches 1024]

MINKOWSKI runs once per order of --orders, each on a column of its own (built, filled and finalized like the others,
then given its order).  F64 columns hold the same synthetic values widened to f64, appended in chunks.

The rows are the library's synthetic f32 rows (append_synthetic), the queries gen_f32 values of another seed.  For each
metric and batch size the two screens alternate in one loop (one warm-up call each first); each rate is the batch over
the median of --reps synchronous calls.  The exact kernel makes one pass over the corpus per query, so its time grows
linearly with the batch: batches above --exact-max are timed at --exact-max queries and scaled (marked "scaled").
Also reported per AUTO row: the library's screen time, fallback / repair counts, the largest candidate set, and the
screen's share of the FP32 issue roof (2 B N D instructions against 33.5 T instr/s: the H100 SXM data-sheet 67 TFLOP/s
counted without FMA; MINKOWSKI counts its order's 2 - 5 instructions per element; none when AUTO ranked the batch with
the exact kernel, as MANHATTAN / CHEBYSHEV do for one query).  Two filtered rows (batch 64): a filter passing 1 % of the rows, and one passing 4000 rows (the
direct regime).  10 queries of the last batch are checked bit for bit against NONE_EXACT.  Prints one JSON line per
row and a summary line; writes them to --out as well.
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

FP32_ISSUE = 33.5e12
# FP32 instructions per (query, row, element): the subtraction, then MANHATTAN's FADD / CHEBYSHEV's FMNMX, or
# MINKOWSKI's multiplication chain and FFMA (screen_lp.cu, minkowski_fma)
INSTR = {"MANHATTAN": 2, "CHEBYSHEV": 2}
MINK_INSTR = {1: 2, 2: 2, 3: 3, 4: 3, 5: 4, 6: 4, 7: 5, 8: 4}


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--batches", default="1,8,32,64,1024")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--exact-max", type=int, default=64)
    ap.add_argument("--metrics", default="MANHATTAN,CHEBYSHEV")
    ap.add_argument("--orders", default="2,3,4,8", help="MINKOWSKI orders")
    ap.add_argument("--dtype", default="F32", choices=["F32", "F64"])
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from surrealdb_b200 import Context, VectorColumn
    from surrealdb_b200.engine import pack_row_filter
    from surrealdb_b200.synthetic import gen_f32

    if not torch.cuda.is_available():
        raise SystemExit("lp_knn_perf.py needs a CUDA device")
    ctx = Context(0)
    batches = [int(b) for b in a.batches.split(",")]
    Qall = gen_f32(0x5DB1, 0, max(batches) * a.dim).reshape(max(batches), a.dim).astype(np.float64)
    lines = []

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        lines.append(line)

    gpu = gpu_info()
    summary = {"config": f"{a.n}x{a.dim} {a.dtype} synthetic", "k": a.k, "gpu": gpu}
    runs = []
    for m in a.metrics.split(","):
        runs += [(m, float(p)) for p in a.orders.split(",")] if m == "MINKOWSKI" else [(m, None)]
    for metric, order in runs:
        col = VectorColumn(ctx, a.dim, metric, a.dtype, capacity=a.n)
        if a.dtype == "F32":
            col.append_synthetic(seed=0x5DB0, first_row=0, n=a.n)
        else:
            step = 250_000
            for r0 in range(0, a.n, step):
                m_ = min(step, a.n - r0)
                col.append(gen_f32(0x5DB0, r0 * a.dim, m_ * a.dim).reshape(m_, a.dim).astype(np.float64))
        col.finalize()
        label = metric
        ins = INSTR.get(metric, 2)
        if order is not None:
            col.set_minkowski_order(order)
            label = f"MINKOWSKI_p{order:g}"
            ins = MINK_INSTR[int(order)]
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
            roof_s = ins * B * a.n * a.dim / FP32_ISSUE
            emit({"metric": label, "dtype": a.dtype, "batch": B, "auto_qps": B / t_a, "exact_qps": B / t_e, "speedup": t_e / t_a,
                  "exact_timed_queries": Be, "exact_scaled": Be != B, "auto_spread_ms": [min(ta) * 1e3, max(ta) * 1e3],
                  "exact_spread_ms": [min(te) * 1e3, max(te) * 1e3], "screen_used": st["screen_used"],
                  "screen_ms": st["screen_ms"], "total_ms": st["total_ms"], "n_fallback": st["n_fallback"],
                  "n_repaired": st["n_repaired"], "max_candidates": st["n_candidates"],
                  "fp32_roof_share": roof_s / (st["screen_ms"] * 1e-3) if st["screen_used"] == 1 else None})
        # filtered batches of 64: 1 % of the rows (screened), 4000 rows (direct regime)
        rng = np.random.default_rng(3)
        Q = Qall[:64]
        mlabel = label
        for label, mask in (("filter_1pct", rng.random(a.n) < 0.01), ("filter_4000_rows", np.zeros(a.n, bool))):
            if label == "filter_4000_rows":
                mask[rng.choice(a.n, 4000, replace=False)] = True
            f = pack_row_filter(mask)
            col.set_screen("AUTO")
            call(col, Q, a.k, filters=f)
            ts = []
            for _ in range(a.reps):
                t, _, st = call(col, Q, a.k, filters=f)
                ts.append(t)
            emit({"metric": mlabel, "batch": 64, "filter": label, "auto_qps": 64 / float(np.median(ts)),
                  "n_passes": st["n_passes"], "screen_ms": st["screen_ms"], "n_fallback": st["n_fallback"]})
        # parity: 10 queries of the last batch, AUTO against the exact kernel, bit for bit
        Qp = Qall[max(batches) - 10:max(batches)]
        col.set_screen("AUTO")
        _, (r_a, d_a, c_a), _ = call(col, Qp, a.k)
        col.set_screen("NONE_EXACT")
        _, (r_e, d_e, c_e), _ = call(col, Qp, a.k)
        summary[f"{mlabel}_parity_10_vs_exact"] = bool(np.array_equal(r_a, r_e) and d_a.tobytes() == d_e.tobytes()
                                                       and np.array_equal(c_a, c_e))
        col.close()
        del col
        torch.cuda.empty_cache()
    emit(summary)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Queries/s of brute-force HAMMING and JACCARD KNN through the count path against the exact kernel.

  python scripts/count_knn_perf.py [--n 10000000 --dim 768 --ks 10,100 --batches 1,8,64,1024 --reps 3 --out x.json]
  python scripts/count_knn_perf.py --dtype F64 --n 5000000 --runs HAMMING:alpha16,JACCARD:alpha16

Columns (generated on the device from a seed with torch, appended from device memory in chunks), --runs METRIC:DATA:
  binary  : 0/1 codes, about a hundred distinct distances over the whole column;
  alpha16 : 16 integer values, the queries from the same alphabet.
For each column, k and batch size three requests alternate in one loop (one warm-up call each first): SIMT_F32 (the
count path, whatever the batch), AUTO (what the library picks: HAMMING ranks a single query with the exact kernel) and
NONE_EXACT (the exact kernel); each rate is the batch over the median of --reps synchronous calls.  The exact kernel
makes one pass over the column per query: batches above --exact-max (JACCARD: --exact-max-jaccard, its exact kernel is
O(D^2) per row) are timed at that many queries and scaled (marked "scaled").  Also reported: the count kernel's
share of the INT32 issue roof (2 B N D instructions -- a compare and an add per element -- against 16.7 T instr/s:
the H100 SXM's 64 INT32 lanes per SM x 132 SMs x 1.98 GHz, computed from shapes, not measured); two filtered rows
(batch 64: a filter passing 1 % of the rows, one passing 4000 rows: the direct regime); 10 queries of the last batch
checked bit for bit against NONE_EXACT; the card's name and power limit, read in the same run.
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

INT32_ISSUE = 64 * 132 * 1.98e9  # HAMMING only: JACCARD's work is binary searches, not a fixed instruction count


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
    ap.add_argument("--ks", default="10,100")
    ap.add_argument("--batches", default="1,8,64,1024")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--exact-max", type=int, default=8)
    ap.add_argument("--exact-max-jaccard", type=int, default=1)
    ap.add_argument("--runs", default="HAMMING:binary,HAMMING:alpha16,JACCARD:alpha16")
    ap.add_argument("--dtype", default="F32", choices=["F32", "F64"])
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from surrealdb_b200 import Context, VectorColumn
    from surrealdb_b200.engine import pack_row_filter

    if not torch.cuda.is_available():
        raise SystemExit("count_knn_perf.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    ctx = Context(0)
    batches = [int(b) for b in a.batches.split(",")]
    ks = [int(k) for k in a.ks.split(",")]
    tdt = torch.float32 if a.dtype == "F32" else torch.float64
    lines = []

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        lines.append(line)

    summary = {"config": f"{a.n}x{a.dim} {a.dtype}", "gpu": gpu_info()}
    for run in a.runs.split(","):
        metric, data = run.split(":")
        hi = 2 if data == "binary" else 16
        g = torch.Generator(device=dev)
        g.manual_seed(0x5DB0 + hi)
        col = VectorColumn(ctx, a.dim, metric, a.dtype, capacity=a.n)
        step = 500_000
        for r0 in range(0, a.n, step):
            m = min(step, a.n - r0)
            chunk = torch.randint(0, hi, (m, a.dim), generator=g, device=dev).to(tdt)
            torch.cuda.synchronize()
            col.append_device(chunk.data_ptr(), m)
            del chunk
        t0 = time.perf_counter()
        col.finalize()
        emit({"metric": metric, "data": data, "finalize_s": time.perf_counter() - t0})
        Qall = torch.randint(0, hi, (max(batches), a.dim), generator=g, device=dev).double().cpu().numpy()
        emax = a.exact_max_jaccard if metric == "JACCARD" else a.exact_max
        for k in ks:
            for B in batches:
                Q = Qall[:B]
                Be = min(B, emax)
                reqs = [("SIMT_F32", Q), ("AUTO", Q), ("NONE_EXACT", Q[:Be])]
                for scr, q in reqs:
                    col.set_screen(scr)
                    call(col, q, k)
                times = {scr: [] for scr, _ in reqs}
                st_count = None
                for _ in range(a.reps):
                    for scr, q in reqs:
                        col.set_screen(scr)
                        t, _, st = call(col, q, k)
                        times[scr].append(t * B / q.shape[0])
                        if scr == "SIMT_F32":
                            st_count = st
                        elif scr == "AUTO":
                            st_auto = st
                med = {scr: float(np.median(v)) for scr, v in times.items()}
                row = {"metric": metric, "data": data, "dtype": a.dtype, "k": k, "batch": B,
                       "count_qps": B / med["SIMT_F32"], "auto_qps": B / med["AUTO"], "exact_qps": B / med["NONE_EXACT"],
                       "count_vs_exact": med["NONE_EXACT"] / med["SIMT_F32"], "exact_timed_queries": Be,
                       "exact_scaled": Be != B, "auto_screen_used": st_auto["screen_used"],
                       "spread_ms": {scr: [min(v) * 1e3, max(v) * 1e3] for scr, v in times.items()},
                       "count_screen_used": st_count["screen_used"], "count_ms": st_count["screen_ms"],
                       "n_fallback": st_count["n_fallback"], "max_candidates": st_count["n_candidates"]}
                if metric == "HAMMING" and st_count["screen_used"] == 1 and st_count["screen_ms"] > 0:
                    sec = st_count["screen_ms"] * 1e-3
                    row["elem_cmp_per_s"] = B * a.n * a.dim / sec
                    row["int32_roof_share"] = 2 * B * a.n * a.dim / INT32_ISSUE / sec
                emit(row)
        rng = np.random.default_rng(3)
        Q = Qall[:64]
        for label, mask in (("filter_1pct", rng.random(a.n) < 0.01), ("filter_4000_rows", np.zeros(a.n, bool))):
            if label == "filter_4000_rows":
                mask[rng.choice(a.n, 4000, replace=False)] = True
            f = pack_row_filter(mask)
            col.set_screen("AUTO")
            call(col, Q, 10, filters=f)
            ts = []
            for _ in range(a.reps):
                t, _, st = call(col, Q, 10, filters=f)
                ts.append(t)
            emit({"metric": metric, "data": data, "batch": 64, "k": 10, "filter": label, "auto_qps": 64 / float(np.median(ts)),
                  "n_passes": st["n_passes"], "n_fallback": st["n_fallback"]})
        Qp = Qall[max(batches) - (2 if metric == "JACCARD" else 10):max(batches)]
        col.set_screen("AUTO")
        _, (r_a, d_a, c_a), _ = call(col, Qp, max(ks))
        col.set_screen("NONE_EXACT")
        _, (r_e, d_e, c_e), _ = call(col, Qp, max(ks))
        summary[f"{metric}_{data}_parity_vs_exact"] = bool(np.array_equal(r_a, r_e) and d_a.tobytes() == d_e.tobytes()
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

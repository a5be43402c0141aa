#!/usr/bin/env python
"""`ORDER BY vector::<fn>(emb, $q) ASC|DESC LIMIT k` on a row-sharded column, measured on one GPU (one rank):

  (a) sdb_corpus_order_sharded_submit + sdb_knn_sharded_wait on a one-rank column (row_base 0) against the unsharded
      sdb_corpus_order_topk on the same column and batch, for vector::similarity::cosine DESC (int8 screen) and
      vector::dot DESC (bf16 screen) on a COSINE column and vector::distance::euclidean DESC on a EUCLIDEAN column;
      host wall time per call and the batch's device time (sdb_knn_last_stats total_ms), and the two results compared
      byte for byte;
  (b) the merge kernel alone (sdb_order_merge_device ASC and DESC, sdb_topk_merge_device) over 8 and 16 emulated
      shard lists of nq queries for several k: host wall time of the synchronous call and the kernel's device time
      from torch.profiler.

  python scripts/sharded_order_perf.py [--n 10000000 --dim 768 --nq 1024 --k 10 --reps 5 --out x.json]

The rows are the library's synthetic rows (append_synthetic), the queries gen_f32 values of another seed.  Every
figure is the median of --reps synchronous calls after one warm-up call.  Several GPUs cannot be measured with one
card; only the one-rank driver and the merge are.  The card's name and power limit are read in the same run.  Prints
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


def timed(fn, reps, stats=None):
    """median host wall ms of fn() after a warm-up call, and (stats given) the median of stats()["total_ms"]"""
    fn()
    ts, ds = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
        if stats:
            ds.append(stats()["total_ms"])
    return float(np.median(ts)), (float(np.median(ds)) if ds else None), [min(ts), max(ts)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--merge-reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from surrealdb_b200 import Context, VectorColumn
    from surrealdb_b200.engine import order_merge_device, topk_merge_device
    from surrealdb_b200.synthetic import gen_f32

    if not torch.cuda.is_available():
        raise SystemExit("sharded_order_perf.py needs a CUDA device")
    ctx = Context(0)
    nq, k = a.nq, a.k
    Q = np.ascontiguousarray(gen_f32(0x5DB1, 0, nq * a.dim).reshape(nq, a.dim).astype(np.float64))
    lines = []

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        lines.append(line)

    summary = {"config": f"{a.n}x{a.dim} F32 synthetic", "k": k, "nq": nq, "gpu": gpu_info(),
               "multi_gpu": "not measured (one card)"}

    # ---- (a) one-rank sharded ORDER BY against the unsharded call ----
    out = (np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64), np.zeros(nq, np.uint32))

    def sharded(col, fn, order):
        t = col.order_sharded_submit_host(Q.ctypes.data, nq, k, fn, order, *(x.ctypes.data for x in out))
        col.sharded_wait(t)
        return out

    for metric, rankings in (("COSINE", (("SIMILARITY_COSINE", "DESC"), ("DOT", "DESC"))),
                             ("EUCLIDEAN", (("EUCLIDEAN", "DESC"),))):
        col = VectorColumn(ctx, a.dim, metric, "F32", capacity=a.n)
        col.append_synthetic(seed=0x5DB0, first_row=0, n=a.n)
        col.finalize()
        col.set_row_base(0)
        for fn, order in rankings:
            ref = col.order_topk(Q, k, fn, order)
            got = sharded(col, fn, order)
            same = all(u.tobytes() == v.tobytes() for u, v in zip(got, ref))
            st = col.stats()
            w_u, d_u, sp_u = timed(lambda: col.order_topk(Q, k, fn, order), a.reps, col.stats)
            w_s, d_s, sp_s = timed(lambda: sharded(col, fn, order), a.reps, col.stats)
            emit({"part": "a", "column": metric, "fn": fn, "order": order, "unsharded_wall_ms": w_u,
                  "unsharded_device_ms": d_u, "unsharded_spread_ms": sp_u, "sharded_wall_ms": w_s,
                  "sharded_device_ms": d_s, "sharded_spread_ms": sp_s, "sharded_over_unsharded_wall": w_s / w_u,
                  "results_identical": same, "screen_used": st["screen_used"], "n_repaired": st["n_repaired"],
                  "n_fallback": st["n_fallback"]})
            summary[f"{metric.lower()}_{fn.lower()}_{order.lower()}_identical"] = same
        col.close()
        del col
        torch.cuda.empty_cache()

    # ---- (b) the merge kernel alone: ASC, DESC and the KNN merge over emulated shard lists ----
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(5)
    for n_lists in (8, 16):
        for kk in (10, 256, 1000, 4096):
            vals = np.sort(rng.standard_normal((n_lists, nq, kk)), axis=-1)
            rows = (np.arange(n_lists, dtype=np.uint64)[:, None, None] * np.uint64(1 << 32)
                    + np.arange(kk, dtype=np.uint64)[None, None, :]) * np.ones((1, nq, 1), np.uint64)
            d_rows = torch.from_numpy(rows.view(np.int64)).to(dev)
            d_asc = torch.from_numpy(vals).to(dev)
            d_desc = torch.from_numpy(np.ascontiguousarray(vals[..., ::-1])).to(dev)
            d_cnt = torch.full((n_lists, nq), kk, dtype=torch.int32, device=dev)
            o = (torch.zeros((nq, kk), dtype=torch.int64, device=dev),
                 torch.zeros((nq, kk), dtype=torch.float64, device=dev), torch.zeros(nq, dtype=torch.int32, device=dev))
            torch.cuda.synchronize()
            po = [t.data_ptr() for t in o]
            calls = {
                "knn": lambda: topk_merge_device(ctx, n_lists, nq, kk, d_rows.data_ptr(), d_asc.data_ptr(),
                                                 d_cnt.data_ptr(), *po),
                "asc": lambda: order_merge_device(ctx, n_lists, nq, kk, "ASC", d_rows.data_ptr(), d_asc.data_ptr(),
                                                  d_cnt.data_ptr(), *po),
                "desc": lambda: order_merge_device(ctx, n_lists, nq, kk, "DESC", d_rows.data_ptr(), d_desc.data_ptr(),
                                                   d_cnt.data_ptr(), *po),
            }
            row = {"part": "b", "n_lists": n_lists, "k": kk, "nq": nq}
            for name, fn in calls.items():
                w, _, sp = timed(fn, a.merge_reps)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(a.merge_reps):
                        fn()
                    torch.cuda.synchronize()
                ev = [e for e in prof.key_averages() if "merge_kernel" in e.key]
                tot = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in ev)
                cnt = sum(e.count for e in ev)
                row[f"{name}_wall_ms"] = w
                row[f"{name}_kernel_us"] = tot / cnt if cnt else "not found in the profile"
            emit(row)
            del d_rows, d_asc, d_desc, d_cnt, o
            torch.cuda.empty_cache()
    emit(summary)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

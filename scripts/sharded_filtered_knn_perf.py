#!/usr/bin/env python
"""Filtered brute-force KNN on a row-sharded column, measured on one GPU (one rank): what slicing the global bitmaps
costs a shard, and what the asynchronous filtered submit with device bitmaps gains over the blocking call.

  python scripts/sharded_filtered_knn_perf.py [--n 10000000 --dim 768 --nq 1024 --k 10 --reps 5 --out x.json]

The column is append_synthetic rows (F32, cosine); queries are corpus rows plus a little noise.  Filters: one random
bitmap per density (100 / 10 / 1 / 0.03 %; the last passes ~3000 rows, the direct regime), shared by the batch.
For each density, alternated --reps times after a warm-up (medians reported):
  filtered        sdb_knn_submit_filtered + wait (host bitmaps of the column's own rows)
  sharded_base0   sdb_knn_sharded_submit_filtered + wait, row_base 0, bitmaps over n rows
  sharded_unal    the same with row_base 1001 inside n + 2002 global rows (an unaligned slice)
each as host wall time (submit to wait) and the batch's device time (sdb_knn_last_stats total_ms).
The slice kernel's device time comes from a separate torch.profiler run (CUDA activities) of the unaligned call;
its bytes and the H2D bytes per batch are computed from the shapes (per rank, R = 1 .. 8).  Then queries/s of
sdb_knn_submit_filtered_device with 1 to 4 tickets in flight (device bitmaps, 10 % density, --batches batches)
against the blocking sdb_knn_bruteforce_filtered_device.  The GPU's name and power limit are printed with the
numbers.  Prints one JSON line; writes it to --out as well.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", type=int, default=16)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from surrealdb_b200 import Context, VectorColumn, pack_row_filter

    ctx = Context(0)
    dev = torch.device("cuda", 0)
    n, nq, k = a.n, a.nq, a.k
    res = {"config": f"{n}x{a.dim} F32 cosine append_synthetic", "nq": nq, "k": k, "gpu": gpu_info()}
    col = VectorColumn(ctx, a.dim, "COSINE", "F32", capacity=n)
    for r0 in range(0, n, 1 << 20):
        col.append_synthetic(11, r0, min(1 << 20, n - r0))
    col.finalize()
    rng = np.random.default_rng(3)
    idx = rng.choice(n, nq, replace=False)
    Q = np.stack([col.read_rows(int(i), 1)[0] for i in idx]).astype(np.float64)
    Q += rng.normal(0, 0.05 * float(np.abs(Q).mean()), Q.shape)
    Q = torch.from_numpy(Q).pin_memory()
    out = [torch.zeros((nq, k), dtype=torch.int64).pin_memory(), torch.zeros((nq, k), dtype=torch.float64).pin_memory(),
           torch.zeros(nq, dtype=torch.int32).pin_memory()]
    o = [t.data_ptr() for t in out]
    lo = 1001  # the unaligned shard: rows [lo, lo + n) of n + 2 lo global rows
    n_unal = n + 2 * lo

    def run(kind, fb):
        col.set_row_base(0 if kind != "sharded_unal" else lo)
        t0 = time.perf_counter()
        if kind == "filtered":
            col.wait(col.submit_host_filtered(Q.data_ptr(), nq, k, fb[kind].data_ptr(), 1, None, *o))
        else:
            total = n if kind == "sharded_base0" else n_unal
            col.sharded_wait(col.sharded_submit_filtered_host(Q.data_ptr(), nq, k, fb[kind].data_ptr(), 1, None, total,
                                                              *o))
        return (time.perf_counter() - t0) * 1e3, col.stats()["total_ms"]

    kinds = ("filtered", "sharded_base0", "sharded_unal")
    words, words_unal = (n + 31) // 32, (n_unal + 31) // 32
    for p in (1.0, 0.1, 0.01, 0.0003):
        m = rng.random(n) < p
        m_unal = np.zeros(n_unal, bool)
        m_unal[lo : lo + n] = m
        fb = {"filtered": torch.from_numpy(pack_row_filter(m).view(np.int32)).pin_memory()}
        fb["sharded_base0"] = fb["filtered"]
        fb["sharded_unal"] = torch.from_numpy(pack_row_filter(m_unal).view(np.int32)).pin_memory()
        name = f"d{p * 100:g}pct"
        ref = None
        for kind in kinds:  # warm-up, and the three calls agree
            run(kind, fb)
            got = [t.numpy().copy() for t in out]
            if kind == "sharded_unal":
                got[0] = got[0] - lo
            if ref is None:
                ref = got
            assert all(np.array_equal(x, y) for x, y in zip(ref, got)), (name, kind)
        res[f"{name}_passing_rows"] = int(m.sum())
        wall = {kd: [] for kd in kinds}
        devt = {kd: [] for kd in kinds}
        for _ in range(a.reps):
            for kind in kinds:
                w, d = run(kind, fb)
                wall[kind].append(w)
                devt[kind].append(d)
        for kind in kinds:
            res[f"{name}_{kind}_wall_ms"] = float(np.median(wall[kind]))
            res[f"{name}_{kind}_device_ms"] = float(np.median(devt[kind]))
        res[f"{name}_direct"] = col.stats()["screen_used"] == 3 and col.stats()["n_passes"] == 0

    # the slice kernel alone: device time from the profiler, bytes from the shapes
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            run("sharded_unal", fb)
        torch.cuda.synchronize()
    sl = [e for e in prof.key_averages() if e.key == "slice_filter_rows_kernel"]
    if sl:
        us = sl[0].device_time_total / max(1, sl[0].count) if hasattr(sl[0], "device_time_total") else \
            sl[0].cuda_time_total / max(1, sl[0].count)
        res["slice_kernel_us"] = float(us)
        res["slice_kernel_bytes"] = 4 * (2 * words + 1)
        res["slice_kernel_GBps"] = res["slice_kernel_bytes"] / (us * 1e-6) / 1e9
    else:
        res["slice_kernel_us"] = "not found in the profile"
    for R in (1, 2, 4, 8):  # H2D bytes per batch and rank: queries + the bitmaps (unsharded: whole; sharded: a span)
        span = min(-(-words // R) + 1, words)
        res[f"h2d_bytes_R{R}"] = {"queries": nq * a.dim * 8, "filters_sharded": 4 * span,
                                  "filters_unsharded_call": 4 * words}

    # asynchronous filtered submits with device bitmaps against the blocking device call
    col.set_row_base(0)
    dq = Q.to(dev)
    dfs = [torch.from_numpy(pack_row_filter(rng.random(n) < 0.1).view(np.int32)).to(dev) for _ in range(4)]
    douts = [(torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64, device=dev),
              torch.zeros(nq, dtype=torch.int32, device=dev)) for _ in range(4)]
    torch.cuda.synchronize()

    def ptrs(i):
        return [t.data_ptr() for t in douts[i]]

    def blocking():
        for b in range(a.batches):
            col.knn_device_filtered(dq.data_ptr(), nq, k, dfs[b % 4].data_ptr(), 1, None, 0, *ptrs(b % 4))

    def in_flight(depth):
        pending = []
        for b in range(a.batches):
            if len(pending) == depth:
                col.wait(pending.pop(0))
            pending.append(col.submit_device_filtered(dq.data_ptr(), nq, k, dfs[b % 4].data_ptr(), 1, None, 0,
                                                      *ptrs(b % 4)))
        for t in pending:
            col.wait(t)

    blocking()
    in_flight(4)
    runs = {"blocking": blocking, **{f"tickets{d}": (lambda d=d: in_flight(d)) for d in (1, 2, 3, 4)}}
    times = {key: [] for key in runs}
    for _ in range(a.reps):
        for key, fn in runs.items():
            t0 = time.perf_counter()
            fn()
            times[key].append(time.perf_counter() - t0)
    for key in runs:
        res[f"device_bitmaps_10pct_{key}_qps"] = a.batches * nq / float(np.median(times[key]))
    col.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

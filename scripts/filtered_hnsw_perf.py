#!/usr/bin/env python
"""Batch-filtered HNSW search (sdb_hnsw_search_filtered_batch_device) on GPU-built 1M-element indexes, against the
single-mask call (sdb_hnsw_search_filtered) where that still succeeds, and the unfiltered walk.

  python scripts/filtered_hnsw_perf.py [--rows 1000000 --dims 128,768 --metrics euclidean,cosine --nq 10000
                                        --k 10 --ef 64 --out filtered_hnsw_perf.json]

Data and graph as `bench_extra.py hnsw --builder incremental` makes them: clustered seeded vectors, build_incremental
(M=16, efc=150) in the walk metric.  Queries: --nq device-resident vectors from the same distribution.  Filters: random
element filters at 100 / 50 / 10 / 5 / 1 / 0.1 / 0 %, a cluster-correlated filter (the elements of 1 % of the clusters),
and 64 distinct random 10 % filters spread over the batch.  A spilled walk can cover the whole reachable layer 0 (at
0 % it does, as the reference's does), so selectivities below --full-below run --nq-small queries instead of --nq.
Per row: queries/s of one timed call after a warm-up call, the share of queries the spill tier finished, mean visited
and expanded elements per query, and the single-mask call's queries/s at the same filter (null where it returns
SDB_EOVERFLOW).  The unfiltered walk (sdb_hnsw_search_device) is timed in the same run for each index.  The GPU's name
and power limit are read in the same run.  Prints one JSON line; writes it to --out as well.
"""
import argparse
import ctypes as C
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
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dims", default="128,768")
    ap.add_argument("--metrics", default="euclidean,cosine")
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--nq-small", type=int, default=512)
    ap.add_argument("--full-below", type=float, default=0.001, help="selectivities below this run --nq-small queries")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--ef", type=int, default=64)
    ap.add_argument("--sigma", type=float, default=0.5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from surrealdb_b200 import Context, HnswIndex
    from surrealdb_b200 import _lib as L
    from surrealdb_b200.hnsw_build import build_incremental
    from surrealdb_b200.engine import pack_row_filter

    ctx = Context(0)
    dev = torch.device("cuda", 0)
    n, k, ef = a.rows, a.k, a.ef
    res = {"rows": n, "nq": a.nq, "nq_small": a.nq_small, "k": k, "ef": ef, "gpu": gpu_info(), "runs": []}
    p = lambda t: C.c_void_p(t.data_ptr())
    for dim in [int(d) for d in a.dims.split(",")]:
        for metric in a.metrics.split(","):
            g = torch.Generator(device=dev).manual_seed(0x5DB00003)
            centers = torch.nn.functional.normalize(torch.randn((4096, dim), generator=g, device=dev), dim=1)
            cl = torch.randint(0, 4096, (n,), generator=g, device=dev)
            x = (centers[cl] + (a.sigma / dim ** 0.5) * torch.randn((n, dim), generator=g, device=dev)).contiguous()
            qc = torch.randint(0, 4096, (a.nq,), generator=g, device=dev)
            queries = (centers[qc] + (a.sigma / dim ** 0.5) * torch.randn((a.nq, dim), generator=g, device=dev)).contiguous()
            t0 = time.perf_counter()
            built = build_incremental(ctx, x, metric.upper(), m=16, m0=32, efc=150, seed=7, growth=0.25)
            torch.cuda.synchronize()
            build_s = time.perf_counter() - t0
            order = built["order"]  # new element id -> original row
            cl_new = cl[torch.as_tensor(order, device=dev).long()].cpu().numpy()
            idx = HnswIndex.from_device(ctx, built["x"], built["layers_dev"], built["entry"], metric.upper())
            del x
            rng = np.random.default_rng(dim + len(metric))

            def call(nq, words, qf, counters=True):
                ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
                dist = torch.empty((nq, k), dtype=torch.float64, device=dev)
                cnt = torch.empty((nq,), dtype=torch.int32, device=dev)
                ctr = torch.empty((2 * nq,), dtype=torch.int64, device=dev)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                L.check(L.lib().sdb_hnsw_search_filtered_batch_device(
                    idx.h, p(queries), nq, k, ef, p(words), words.shape[0],
                    None if qf is None else C.c_void_p(qf.ctypes.data), p(ids), p(dist), p(cnt), p(ctr)))
                dt = time.perf_counter() - t0
                c = ctr.view(nq, 2).double().mean(0).tolist()
                return nq / dt, idx.last_spilled() / nq, c

            def old_rate(nq, mask):
                qh = queries[:nq].cpu().numpy()
                t = np.ascontiguousarray(mask, np.uint8)
                ids, dist = np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float64)
                cnt = np.zeros(nq, np.uint32)
                st = L.lib().sdb_hnsw_search_filtered(idx.h, C.c_void_p(qh.ctypes.data), nq, k, ef, C.c_void_p(t.ctypes.data),
                                                      C.c_void_p(ids.ctypes.data), C.c_void_p(dist.ctypes.data),
                                                      C.c_void_p(cnt.ctypes.data), None)
                if st != L.SDB_OK:
                    return None
                t0 = time.perf_counter()
                L.check(L.lib().sdb_hnsw_search_filtered(idx.h, C.c_void_p(qh.ctypes.data), nq, k, ef, C.c_void_p(t.ctypes.data),
                                                         C.c_void_p(ids.ctypes.data), C.c_void_p(dist.ctypes.data),
                                                         C.c_void_p(cnt.ctypes.data), None))
                return nq / (time.perf_counter() - t0)  # host variant: includes the copies of queries and mask

            rows = []
            filters = [(f"random {s * 100:g} %", s, (rng.random(n) < s)[None, :], None) for s in (1.0, 0.5, 0.1, 0.05, 0.01, 0.001, 0.0)]
            picked = rng.choice(4096, 41, replace=False)
            filters.append(("cluster-correlated 1 % of clusters", 0.01, np.isin(cl_new, picked)[None, :], None))
            many = rng.random((64, n)) < 0.1
            filters.append(("64 distinct 10 % filters", 0.1, many, None))
            for name, s, masks, _ in filters:
                nq = a.nq if s >= a.full_below else a.nq_small
                qf = (np.arange(nq) % masks.shape[0]).astype(np.uint32) if masks.shape[0] > 1 else None
                words = torch.from_numpy(pack_row_filter(masks)).to(dev)
                call(min(nq, 256), words, None if qf is None else qf[:256])  # warm-up
                qps, spill, (vis, exp) = call(nq, words, qf)
                row = {"filter": name, "nq": nq, "qps": round(qps), "spilled": round(spill, 4),
                       "visited_per_q": round(vis, 1), "expanded_per_q": round(exp, 1),
                       "single_mask_qps": None if masks.shape[0] > 1 else old_rate(nq, masks[0])}
                if row["single_mask_qps"] is not None:
                    row["single_mask_qps"] = round(row["single_mask_qps"])
                rows.append(row)
                print(json.dumps({"dim": dim, "metric": metric, **row}), file=sys.stderr, flush=True)
            # the unfiltered walk on the same index and queries
            ids = torch.empty((a.nq, k), dtype=torch.int64, device=dev)
            dist = torch.empty((a.nq, k), dtype=torch.float64, device=dev)
            cnt = torch.empty((a.nq,), dtype=torch.int32, device=dev)
            unf = []
            for _ in range(4):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                L.check(L.lib().sdb_hnsw_search_device(idx.h, p(queries), a.nq, k, ef, p(ids), p(dist), p(cnt)))
                unf.append(a.nq / (time.perf_counter() - t0))
            res["runs"].append({"dim": dim, "metric": metric, "build_s": round(build_s, 1),
                                "unfiltered_qps": round(float(np.median(unf[1:]))), "rows": rows})
            idx.close()
            del built, idx, queries
            torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Asynchronous HNSW tickets (sdb_hnsw_submit[_device], sdb_hnsw_submit_filtered[_device] + sdb_hnsw_wait) against
back-to-back blocking calls on the same GPU-built 1M-element indexes.

  python scripts/hnsw_submit_perf.py [--rows 1000000 --dims 128,768 --metrics euclidean,cosine --batches 64,256,1024
                                      --k 10 --ef 64 --rounds 3 --out hnsw_submit_perf.json]

Data and graph as `scripts/filtered_hnsw_perf.py` makes them: clustered seeded vectors, build_incremental (M=16,
efc=150) in the walk metric.  For every batch size, with the queries and outputs in pinned host memory and on the device,
and for three cases (unfiltered, one random 10 % filter, one random 1 % filter, whose queries mostly spill), a stream of
batches runs three ways: blocking calls back to back, and tickets with 2 and with 4 in flight (submit batch i, wait for
batch i - depth).  The three alternate, --rounds times; the figure is the median queries/s.  Every ticket's outputs
are compared with the blocking call's (counts, counters and each row's first count entries).  The GPU's name and
power limit are read in the same run.  Prints one JSON line; writes it to --out as well.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from collections import deque

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
    ap.add_argument("--batches", default="64,256,1024")
    ap.add_argument("--queries", type=int, default=8192, help="queries per timed stream (at least 8 batches)")
    ap.add_argument("--queries-spill", type=int, default=2048, help="the same for the 1 %% filter")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--ef", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sigma", type=float, default=0.5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from surrealdb_b200 import Context, HnswIndex
    from surrealdb_b200 import _lib as L
    from surrealdb_b200.engine import pack_row_filter
    from surrealdb_b200.hnsw_build import build_incremental

    lib = L.lib()
    ctx = Context(0)
    dev = torch.device("cuda", 0)
    n, k, ef = a.rows, a.k, a.ef
    res = {"rows": n, "k": k, "ef": ef, "rounds": a.rounds, "gpu": gpu_info(), "runs": []}
    ptr = lambda t: C.c_void_p(t.data_ptr())
    batches = [int(b) for b in a.batches.split(",")]
    q_max = max(max(8 * b, a.queries) for b in batches)
    for dim in [int(d) for d in a.dims.split(",")]:
        for metric in a.metrics.split(","):
            g = torch.Generator(device=dev).manual_seed(0x5DB00003)
            centers = torch.nn.functional.normalize(torch.randn((4096, dim), generator=g, device=dev), dim=1)
            cl = torch.randint(0, 4096, (n,), generator=g, device=dev)
            x = (centers[cl] + (a.sigma / dim ** 0.5) * torch.randn((n, dim), generator=g, device=dev)).contiguous()
            qc = torch.randint(0, 4096, (q_max,), generator=g, device=dev)
            d_q = (centers[qc] + (a.sigma / dim ** 0.5) * torch.randn((q_max, dim), generator=g, device=dev)).contiguous()
            h_q = d_q.cpu().pin_memory()
            built = build_incremental(ctx, x, metric.upper(), m=16, m0=32, efc=150, seed=7, growth=0.25)
            idx = HnswIndex.from_device(ctx, built["x"], built["layers_dev"], built["entry"], metric.upper())
            del x
            rng = np.random.default_rng(dim + len(metric))
            h = idx.h
            cases = [("unfiltered", None), ("10 %", rng.random(n) < 0.1), ("1 %", rng.random(n) < 0.01)]
            for case, mask in cases:
                words_h = None if mask is None else torch.from_numpy(pack_row_filter(mask[None, :])).pin_memory()
                words_d = None if mask is None else words_h.to(dev)
                for B in batches:
                    nb = max(8, (a.queries_spill if case == "1 %" else a.queries) // B)
                    for where in ("pinned host", "device"):
                        on_dev = where == "device"
                        mk = (lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)) if on_dev else \
                            (lambda shape, dt: torch.empty(shape, dtype=dt).pin_memory())
                        outs = {m: [(mk((B, k), torch.int64), mk((B, k), torch.float64), mk((B,), torch.int32),
                                     mk((2 * B,), torch.int64)) for _ in range(nb)] for m in ("blocking", "tickets")}
                        qsrc = d_q if on_dev else h_q
                        words = words_d if on_dev else words_h

                        def qp(i):
                            return C.c_void_p(qsrc.data_ptr() + i * B * dim * 4)

                        def blocking(i, o):
                            if mask is None and on_dev:  # (no counters in the blocking device call)
                                return lib.sdb_hnsw_search_device(h, qp(i), B, k, ef, ptr(o[0]), ptr(o[1]), ptr(o[2]))
                            if mask is None:
                                return lib.sdb_hnsw_search(h, qp(i), B, k, ef, *map(ptr, o))
                            f = lib.sdb_hnsw_search_filtered_batch_device if on_dev else lib.sdb_hnsw_search_filtered_batch
                            return f(h, qp(i), B, k, ef, ptr(words), 1, None, *map(ptr, o))

                        def submit(i, o, t):
                            if mask is None and on_dev:
                                return lib.sdb_hnsw_submit_device(h, qp(i), B, k, ef, ptr(o[0]), ptr(o[1]), ptr(o[2]),
                                                                  None, C.byref(t))
                            if mask is None:
                                return lib.sdb_hnsw_submit(h, qp(i), B, k, ef, None, *map(ptr, o), C.byref(t))
                            f = lib.sdb_hnsw_submit_filtered_device if on_dev else lib.sdb_hnsw_submit_filtered
                            return f(h, qp(i), B, k, ef, ptr(words), 1, None, *map(ptr, o), C.byref(t))

                        def run(mode):
                            torch.cuda.synchronize()
                            t0 = time.perf_counter()
                            if mode == "blocking":
                                for i in range(nb):
                                    L.check(blocking(i, outs["blocking"][i]))
                            else:
                                depth = int(mode.split()[0])
                                inflight = deque()
                                for i in range(nb):
                                    if len(inflight) == depth:
                                        L.check(lib.sdb_hnsw_wait(h, inflight.popleft()))
                                    t = C.c_uint32()
                                    L.check(submit(i, outs["tickets"][i], t))
                                    inflight.append(t.value)
                                while inflight:
                                    L.check(lib.sdb_hnsw_wait(h, inflight.popleft()))
                            torch.cuda.synchronize()
                            return nb * B / (time.perf_counter() - t0)

                        modes = ["blocking", "2 tickets", "4 tickets"]
                        for m in modes:  # warm-up: every shape, every buffer
                            run(m)
                        rates = {m: [] for m in modes}
                        for _ in range(a.rounds):
                            for m in modes:
                                rates[m].append(run(m))
                        same = True
                        for ob, ot in zip(outs["blocking"], outs["tickets"]):
                            b = [t.cpu().numpy() for t in ob]
                            t = [t.cpu().numpy() for t in ot]
                            n_ctr = 0 if (mask is None and on_dev) else 2 * B
                            same &= b[2].tobytes() == t[2].tobytes() and b[3][:n_ctr].tobytes() == t[3][:n_ctr].tobytes()
                            for r, c in enumerate(b[2].tolist()):
                                same &= b[0][r, :c].tobytes() == t[0][r, :c].tobytes()
                                same &= b[1][r, :c].tobytes() == t[1][r, :c].tobytes()
                        row = {"dim": dim, "metric": metric, "case": case, "batch": B, "queries": where,
                               "batches": nb, "same_outputs": bool(same)}
                        for m in modes:
                            row[m.replace(" ", "_") + "_qps"] = round(float(np.median(rates[m])))
                        res["runs"].append(row)
                        print(json.dumps(row), file=sys.stderr, flush=True)
                        del outs
            idx.close()
            del built, idx, d_q, h_q
            torch.cuda.empty_cache()
    res["all_same"] = all(r["same_outputs"] for r in res["runs"])
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

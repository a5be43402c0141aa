#!/usr/bin/env python
"""Times batches of documents through one graph call (sdb_graph_expand_batch_device, sdb_graph_collect_batch) on the C5
graph shape of graph_filter_perf.py: R-MAT (a,b,c,d = .57,.19,.19,.05), 50M nodes, 500M edges.

  python scripts/graph_batch_perf.py [--nodes 50000000 --edges 500000000 --docs 1,64,1024,16384
                                      --collect-docs 1,64,1024 --reps 5 --out graph_batch_perf.json]

Every document is one random source with out-edges.  Each figure is the median of --reps CUDA-event timings on the
library's stream after a warm-up:
  expand           3 hops, limit 32: the batch call, the flat call on the same frontier (what the document offsets
                   cost), and a loop of single-document calls (ms per document, over at most 256 documents)
  filtered expand  the same with a 50 % edge bitmap, at limit 32 over 3 hops and at limit 0 over 2 hops (where the batch
                   hop counts passing candidates per source and the flat hop per block)
  collect          {1..3+collect} (large reaches on C5) and {1..1+collect} (small ones): the batch call against a loop
                   of sdb_graph_collect (ms per document, at most 256), with the pair table's peak bytes, its growths,
                   the level passes repeated after an overflow and the runs of documents split in two
The outputs are checked inside the script: the batch output against the flat call, and each looped document against
its segment.  Prints one JSON line with the card's name and power limit; writes it to --out as well.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from graph_filter_perf import DevIds, device_bits, gpu_info, rmat_csr  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=50_000_000)
    ap.add_argument("--edges", type=int, default=500_000_000)
    ap.add_argument("--docs", default="1,64,1024,16384")
    ap.add_argument("--collect-docs", default="1,64,1024")
    ap.add_argument("--collect-depths", default="3,1", help="max_depth of the {1..max+collect} runs")
    ap.add_argument("--loop-max", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import torch
    from surrealdb_b200 import Context, SdbError
    from surrealdb_b200.graph import (CsrGraph, collect, collect_batch, device_free, expand_batch_device, expand_device,
                                      expand_filtered_device, last_collect_table)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = Context(0)
    st = torch.cuda.ExternalStream(ctx.stream())
    t0 = time.perf_counter()
    rp, ci = rmat_csr(a.nodes, a.edges, dev, 0x5DB00005)
    graph = CsrGraph(ctx, rp, ci)
    gen_s = time.perf_counter() - t0
    deg = np.diff(rp.astype(np.int64))
    pool = np.nonzero(deg > 0)[0]
    rng = np.random.default_rng(11)
    eb50 = device_bits(ci.size, 0.5, dev, torch.Generator(device=dev).manual_seed(7))
    torch.cuda.synchronize()

    def timed(fn, free=True):
        """median ms of fn() (CUDA events on the library's stream; every call ends synchronised with the host)"""
        r = fn()
        if free:
            device_free(ctx, r[0])
        ms = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            r = fn()
            e1.record(st)
            e1.synchronize()
            if free:
                device_free(ctx, r[0])
            ms.append(e0.elapsed_time(e1))
        return float(np.median(ms))

    def d2h(ptr, n):
        return torch.as_tensor(DevIds(ptr, n), device=dev).cpu().numpy().view(np.uint32) if n else np.zeros(0, np.uint32)

    expand_rows = []
    for n_docs in [int(x) for x in a.docs.split(",") if x]:
        src = rng.choice(pool, n_docs).astype(np.uint32)
        d_src = torch.from_numpy(src.view(np.int32)).to(dev)
        d_off = torch.arange(n_docs + 1, dtype=torch.int64, device=dev)
        d_out_off = torch.zeros(n_docs + 1, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        for name, filt, limit, n_hops in (("unfiltered", None, 32, 3), ("edge 50%", (eb50, None), 32, 3),
                                          ("edge 50%", (eb50, None), 0, 2)):
            hops = [graph] * n_hops
            filters = None if filt is None else [filt] * n_hops

            def batch():
                return expand_batch_device(ctx, hops, d_src.data_ptr(), n_docs, d_off.data_ptr(), n_docs,
                                           d_out_off.data_ptr(), limit, filters)

            def flat():
                if filters is None:
                    return expand_device(ctx, hops, d_src.data_ptr(), n_docs, limit)
                return expand_filtered_device(ctx, hops, filters, d_src.data_ptr(), n_docs, limit)
            row = {"config": name, "limit": limit, "hops": n_hops, "docs": n_docs}
            try:
                row["batch_ms"] = timed(batch)
                row["flat_ms"] = timed(flat)
            except SdbError as e:  # an unlimited chain may exceed 2^32 ids
                row["error"] = str(e)
                expand_rows.append(row)
                continue
            ptr, n = batch()
            got, off = d2h(ptr, n), d_out_off.cpu().numpy().view(np.uint64).copy()
            device_free(ctx, ptr)
            ptr, n_flat = flat()
            assert n_flat == n and np.array_equal(d2h(ptr, n_flat), got), "batch != flat"
            device_free(ctx, ptr)
            n_loop = min(n_docs, a.loop_max)

            def loop():
                last = None
                for d in range(n_loop):
                    if last:
                        device_free(ctx, last)
                    p = d_src.data_ptr() + 4 * d
                    last = (expand_device(ctx, hops, p, 1, limit) if filters is None else
                            expand_filtered_device(ctx, hops, filters, p, 1, limit))[0]
                return last, 0
            row["loop_ms_per_doc"] = timed(loop) / n_loop
            for d in range(0, n_loop, max(1, n_loop // 16)):
                p = d_src.data_ptr() + 4 * d
                ptr, m = (expand_device(ctx, hops, p, 1, limit) if filters is None else
                          expand_filtered_device(ctx, hops, filters, p, 1, limit))
                assert np.array_equal(d2h(ptr, m), got[int(off[d]):int(off[d + 1])]), ("doc", d)
                device_free(ctx, ptr)
            row["results"] = int(n)
            row["batch_ms_per_doc"] = row["batch_ms"] / n_docs
            row["offsets_cost"] = row["batch_ms"] / row["flat_ms"] - 1.0
            expand_rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)

    collect_rows = []
    for mx, n_docs in [(int(m), int(x)) for m in a.collect_depths.split(",") for x in a.collect_docs.split(",") if x]:
        src = rng.choice(pool, n_docs).astype(np.uint32)
        docs = [src[d:d + 1] for d in range(n_docs)]
        row = {"docs": n_docs, "min_depth": 1, "max_depth": mx}
        try:
            row["batch_ms"] = timed(lambda: (collect_batch(graph, docs, 1, mx, False), 0), free=False)
        except SdbError as e:
            row["error"] = str(e)
            collect_rows.append(row)
            continue
        got = collect_batch(graph, docs, 1, mx, False)
        diag = last_collect_table(graph)
        row["table_peak_bytes"], row["table_grows"] = diag["peak_bytes"], diag["grows"]
        row["repeated_passes"], row["document_splits"] = diag["repeated_passes"], diag["splits"]
        row["results"] = int(sum(x.size for x in got))
        n_loop = min(n_docs, a.loop_max)
        row["loop_ms_per_doc"] = timed(lambda: ([collect(graph, docs[d], 1, mx, False) for d in range(n_loop)], 0),
                                       free=False) / n_loop
        for d in range(0, n_loop, max(1, n_loop // 16)):
            assert np.array_equal(collect(graph, docs[d], 1, mx, False), got[d]), ("collect doc", d)
        row["batch_ms_per_doc"] = row["batch_ms"] / n_docs
        collect_rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)

    res = {"bench": "graph_batch_perf", "gpu": gpu_info(),
           "graph": {"nodes": a.nodes, "edges_unique": int(ci.size), "max_degree": int(deg.max()), "generation_s": gen_s},
           "reps": a.reps, "timing": "median of reps, CUDA events", "expand": expand_rows, "collect": collect_rows}
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()

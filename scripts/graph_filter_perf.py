#!/usr/bin/env python
"""Times the WHERE-filtered hop (sdb_graph_expand_filtered_device) against the unfiltered one (sdb_graph_expand_device)
on the C5 graph shape: R-MAT (a,b,c,d = .57,.19,.19,.05), 50M nodes, 500M edges, 3 hops from 1024 sources with the
per-source limit 32 that bench_extra.py graph uses (without it the third level exceeds 2^32 ids).

  python scripts/graph_filter_perf.py [--nodes 50000000 --edges 500000000 --sources 1024 --hops 3
                                       --limit 32 --reps 5 --out graph_filter_perf.json]

Every hop is timed on its own (CUDA events on the library's stream around one device-resident call, median of --reps
after a warm-up), so each filtered hop is compared with the unfiltered hop over the SAME frontier.  Configurations: no
filter; edge bitmaps of density 100 %, 50 % and 1 %; the same each with a 50 % target bitmap.  Effective bandwidth uses
the algorithmic bytes of a hop over F sources with T candidate edges (the unfiltered hop's size without a limit) and
W results:
  unfiltered  16F + 8W                     (row_ptr pair per source, col_idx read and result written per result)
  filtered    16F + 4T + T/8 [edge bits] + 4T [one target word per candidate] + 4W
Prints one JSON line; writes it to --out as well.
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


class DevIds:
    """n uint32 ids at a device pointer, as torch sees them (__cuda_array_interface__)"""
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3}


def rmat_csr(n_nodes, n_edges, dev, seed):
    """R-MAT edges generated on the GPU, one edge per (src, dst), rows in (src, dst) order -> host (row_ptr, col_idx)"""
    import torch
    g = torch.Generator(device=dev).manual_seed(seed)
    bits = max(1, int(np.ceil(np.log2(n_nodes))))
    keys, chunk = [], 1 << 27
    for e0 in range(0, n_edges, chunk):
        ne = min(chunk, n_edges - e0)
        src = torch.zeros(ne, dtype=torch.int64, device=dev)
        dst = torch.zeros(ne, dtype=torch.int64, device=dev)
        for _ in range(bits):
            r = torch.rand(ne, generator=g, device=dev)
            src = (src << 1) | (r >= 0.76).long()
            dst = (dst << 1) | (((r >= 0.57) & (r < 0.76)) | (r >= 0.95)).long()
        keys.append((src % n_nodes) * n_nodes + dst % n_nodes)
        del src, dst, r
    key = torch.unique(torch.cat(keys))
    del keys
    src, dst = key // n_nodes, key % n_nodes
    del key
    row_ptr = torch.zeros(n_nodes + 1, dtype=torch.int64, device=dev)
    row_ptr[1:] = torch.cumsum(torch.bincount(src, minlength=n_nodes), 0)
    del src
    rp = row_ptr.cpu().numpy().astype(np.uint64)
    ci = dst.to(torch.int32).cpu().numpy().view(np.uint32)
    del row_ptr, dst
    torch.cuda.empty_cache()
    return rp, ci


def device_bits(n, density, dev, gen):
    """ceil(n / 32) packed words with each bit set with probability `density`, on the device (int32 tensor)"""
    import torch
    words = (n + 31) // 32
    if density >= 1.0:
        return torch.full((words,), -1, dtype=torch.int32, device=dev)
    if density == 0.5:
        return torch.randint(-(1 << 31), 1 << 31, (words,), generator=gen, dtype=torch.int64, device=dev).to(torch.int32)
    out = torch.empty(words, dtype=torch.int32, device=dev)
    weights = (torch.ones(32, dtype=torch.int64, device=dev) << torch.arange(32, device=dev))
    step = 1 << 22
    for w0 in range(0, words, step):
        w1 = min(words, w0 + step)
        m = torch.rand((w1 - w0, 32), generator=gen, device=dev) < density
        v = (m.long() * weights).sum(1)
        out[w0:w1] = torch.where(v >= 1 << 31, v - (1 << 32), v).to(torch.int32)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=50_000_000)
    ap.add_argument("--edges", type=int, default=500_000_000)
    ap.add_argument("--sources", type=int, default=1024)
    ap.add_argument("--hops", type=int, default=3)
    ap.add_argument("--limit", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import torch
    from surrealdb_b200 import Context
    from surrealdb_b200.graph import CsrGraph, device_free, expand_device, expand_filtered_device
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = Context(0)
    st = torch.cuda.ExternalStream(ctx.stream())
    t0 = time.perf_counter()
    rp, ci = rmat_csr(a.nodes, a.edges, dev, 0x5DB00005)
    graph = CsrGraph(ctx, rp, ci)
    gen_s = time.perf_counter() - t0
    deg = np.diff(rp.astype(np.int64))
    sources = np.random.default_rng(11).choice(np.nonzero(deg > 0)[0], a.sources, replace=False).astype(np.uint32)
    d_src = torch.from_numpy(sources.view(np.int32)).to(dev)
    gen = torch.Generator(device=dev).manual_seed(7)
    configs = [("none", None, None)]
    for ed in (1.0, 0.5, 0.01):
        configs.append((f"edge {ed:.0%}", ed, None))
    for ed in (1.0, 0.5, 0.01):
        configs.append((f"edge {ed:.0%} + target 50%", ed, 0.5))

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        device_free(ctx, fn()[0])  # warm-up
        ms = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            e0.record(st)
            ptr, n = fn()
            e1.record(st)
            e1.synchronize()
            device_free(ctx, ptr)
            ms.append(e0.elapsed_time(e1))
        return float(np.median(ms)), ms

    results = []
    for name, ed, td in configs:
        eb = None if ed is None else device_bits(ci.size, ed, dev, gen)
        tb = None if td is None else device_bits(rp.size - 1, td, dev, gen)
        torch.cuda.synchronize()
        filt = None if eb is None and tb is None else (eb, tb)
        hops = []
        ptr, n = d_src.data_ptr(), sources.size
        owned = None
        for h in range(a.hops):
            def unfiltered(ptr=ptr, n=n, lim=a.limit):
                return expand_device(ctx, [graph], ptr, n, lim)
            def filtered(ptr=ptr, n=n):
                return expand_filtered_device(ctx, [graph], [filt], ptr, n, a.limit)
            fr = torch.as_tensor(DevIds(ptr, n), device=dev).cpu().numpy().view(np.uint32)
            T = int(deg[fr].sum())  # candidate edges: the hop's size without a limit (may exceed 2^32)
            ms_u, _ = timed(unfiltered)
            up, W_u = unfiltered()
            if filt is None:
                ms_f, W, nxt = ms_u, W_u, up
            else:
                device_free(ctx, up)
                ms_f, _ = timed(filtered)
                nxt, W = filtered()
            b_u = 16.0 * n + 8.0 * W_u
            b_f = 16.0 * n + 4.0 * T + (T / 8.0 if eb is not None else 0) + (4.0 * T if tb is not None else 0) + 4.0 * W
            hops.append({"frontier": int(n), "candidates": int(T), "results": int(W), "unfiltered_results": int(W_u),
                         "ms": ms_f, "unfiltered_ms": ms_u, "overhead_vs_unfiltered": ms_f / ms_u - 1.0,
                         "bytes": b_f if filt else b_u, "gbs": (b_f if filt else b_u) / (ms_f * 1e-3) / 1e9,
                         "unfiltered_gbs": b_u / (ms_u * 1e-3) / 1e9})
            if owned:
                device_free(ctx, owned)
            owned, ptr, n = nxt, nxt, W
            if n == 0:
                break
        if owned:
            device_free(ctx, owned)
        results.append({"config": name, "hops": hops, "total_ms": sum(h["ms"] for h in hops)})
        del eb, tb
        torch.cuda.empty_cache()
    res = {"bench": "graph_filter_perf", "gpu": gpu_info(),
           "graph": {"nodes": a.nodes, "edges_unique": int(ci.size), "max_degree": int(deg.max()), "generation_s": gen_s,
                     "shape": "R-MAT (.57,.19,.19,.05), one edge per (src, dst), rows in (src, dst) order"},
           "sources": a.sources, "per_source_limit": a.limit, "reps": a.reps, "timing": "median of reps, CUDA events",
           "results": results}
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()

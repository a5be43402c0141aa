"""A/B of the brute-force pipeline at the 8-GPU shard size (1.25M x 768, B = 1024, k = 10) on ONE GPU:
python scripts/shard_perf.py [rows]   -> one line per configuration (same box, same process)"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from surrealdb_b200 import Context, VectorColumn
from surrealdb_b200.synthetic import gen_f32

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 1_250_000
dim, nq, k, nb = 768, 1024, 10, 24
ctx = Context(0)
dev = torch.device("cuda", 0)
col = VectorColumn(ctx, dim, "COSINE", "F32", capacity=rows)
for r0 in range(0, rows, 1 << 20):
    col.append_synthetic(0x5DB00002, r0, min(1 << 20, rows - r0))
col.finalize()
qs = [torch.from_numpy(gen_f32(0x5DB0A000 + b, 0, nq * dim).reshape(nq, dim).astype(np.float64)).to(dev) for b in range(nb)]
outs = [(torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64, device=dev),
         torch.zeros((nq,), dtype=torch.int32, device=dev)) for _ in range(2)]
stream = torch.cuda.ExternalStream(ctx.stream(), device=dev)
torch.cuda.synchronize()


def run(label, schedule=True, screen="AUTO", depth=2):
    col.set_schedule(schedule)
    col.set_screen(screen)
    def loop(first, last, stats):
        pend = []
        for b in range(first, last):
            o = outs[b % 2]
            pend.append(col.submit_device(qs[b].data_ptr(), nq, k, 0, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr()))
            if len(pend) == depth:
                col.wait(pend.pop(0)); stats.append(col.stats())
        while pend:
            col.wait(pend.pop(0)); stats.append(col.stats())
    loop(0, 4, [])
    torch.cuda.synchronize()
    best = None
    for rep in range(3):
        st = []
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        loop(4, nb, st)
        e1.record(stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / (nb - 4)
        best = ms if best is None or ms < best else best
    scr = np.mean([s["screen_ms"] for s in st]); tot = np.mean([s["total_ms"] for s in st])
    print(f"{label:34s} step {best:7.3f} ms  lib_total {tot:6.3f}  screen {scr:6.3f}  tail {tot-scr:6.3f}  surv/q {np.mean([s['n_survivors'] for s in st])/nq:7.1f}"
          f"  rerank/q {np.mean([s['n_reranked'] for s in st])/nq:6.1f}  passes {st[-1]['n_passes']} fb {sum(s['n_fallback'] for s in st)}", flush=True)


run("streaming, 2 streams (default)")
run("2 streams depth 3", depth=3)
run("2 streams depth 1", depth=1)
run("multipass", schedule=False)
run("streaming, 2 streams again")

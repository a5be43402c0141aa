"""Fingerprints of the graphs the F32 COSINE / EUCLIDEAN builders make on finite data with fixed seeds, so that two
versions of the builder can be shown to make byte-identical graphs (changes to hnsw_select_kernel or to the builders'
handling of NaN distances must not change them).

  python scripts/select_graph_parity.py [--tree DIR] [--out file.json]

prints one line per (builder, metric, shape): the SHA-256 of every layer's row_ptr and col_idx, the entry point and
the edge count.  --tree: import surrealdb_b200 (and its built library) from another checkout, e.g. an older commit
extracted with `git archive` and built; run once per tree and compare the outputs."""
import argparse
import hashlib
import json
import os
import sys

import numpy as np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="the checkout to import surrealdb_b200 from (default: this one)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.tree))
    import torch
    from surrealdb_b200 import Context
    from surrealdb_b200.hnsw_build import build_incremental, build_layers
    ctx = Context(0)
    res = {}
    for metric in ("COSINE", "EUCLIDEAN"):
        for n, dim, seed in ((20000, 64, 1), (6000, 768, 2)):
            rng = np.random.default_rng(seed)
            c = rng.integers(0, 40, n)
            x = (rng.normal(0, 1, (40, dim))[c] + 0.3 * rng.normal(0, 1, (n, dim))).astype(np.float32)
            xd = torch.from_numpy(x).cuda()
            layers, entry, _ = build_layers(ctx, xd, n, dim, metric, m=16, m0=32, seed=seed)
            inc = build_incremental(ctx, xd, metric, m=16, m0=32, efc=100, seed=seed, boot_min=2000)
            inc_layers = [(rp.cpu().numpy().astype(np.uint64), ci.cpu().numpy().astype(np.uint32)[: int(rp[-1])])
                          for rp, ci in inc["layers_dev"]]
            for name, lay, ep in (("layers", layers, entry), ("incremental", inc_layers, inc["entry"])):
                h = hashlib.sha256()
                for rp, ci in lay:
                    h.update(np.ascontiguousarray(rp, np.uint64).tobytes())
                    h.update(np.ascontiguousarray(ci, np.uint32).tobytes())
                key = f"{name} {metric} n={n} dim={dim}"
                res[key] = {"sha256": h.hexdigest(), "entry": int(ep), "edges": int(sum(int(rp[-1]) for rp, _ in lay))}
                print(key, res[key], flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""GPU_CAGRA build with the exact intermediate graph against build_algo NN_DESCENT (DESIGN §4.12, §6):

  --rows x 128 datagen.clustered (L2), nq 10000, k 10, intermediate_graph_degree 128, graph_degree 64

For each build: wall time, and build_ms split into graph / prune / merge (CUDA events, from the index meta).  For
NN-descent: the iterations run and updates(t) (kb2_debug_cagra_knn_graph), and the recall of G0 on --sample rows
against a FLAT search with k = m + 1 (the row itself dropped).  For both graphs, at itopk_size {32, 64, 128} x
search_width {1, 4}: recall@10 against the exact FLAT search and queries/s (median device time of --reps batches after a
warm-up, CUDA events).  --no-exact skips the exact build (at 10M rows it is quadratic).  The card name and power limit
are read in the same run.  Prints one JSON line.

  python scripts/bench_cagra_nn_descent.py [--rows 1000000] [--no-exact] [--nq 10000] [--reps 5] [--sample 10000]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402

from bench_cagra import recall, timed  # noqa: E402
from bench_large_k import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--no-exact", action="store_true")
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=10000)
    args = ap.parse_args()
    import torch

    import knowhere_b200 as kb
    from knowhere_b200 import datagen
    n, d, k, igd, gd = args.rows, 128, 10, 128, 64
    m = min(igd, n - 1)
    dev = torch.device("cuda", 0)
    xb = datagen.clustered(n, d, 42)
    xq = datagen.clustered(args.nq, d, 43)
    gpu, power = card()
    res = {"gpu": gpu, "power_limit_w": power, "rows": n, "dim": d, "nq": args.nq, "k": k,
           "intermediate_graph_degree": igd, "graph_degree": gd}
    xb_d = torch.from_numpy(xb).to(dev)
    xq_d = torch.from_numpy(xq).to(dev)
    flat = kb.Index("FLAT", "L2", d)
    flat.add(xb_d)
    gt = flat.search(xq_d, k)[0].cpu().numpy()
    rows = np.sort(np.random.default_rng(0).choice(n, min(args.sample, n), replace=False))
    g0_gt = flat.search(xb_d[torch.from_numpy(rows).to(dev)], m + 1)[0].cpu().numpy()
    del flat

    builds = [("nn_descent", {"build_algo": "NN_DESCENT"})]
    if not args.no_exact:
        builds.insert(0, ("exact", {}))
    for name, extra in builds:
        torch.cuda.synchronize()
        t0 = time.time()
        ix = kb.Index("GPU_CAGRA", "L2", d, dict(extra, intermediate_graph_degree=igd, graph_degree=gd))
        ix.build(xb_d)
        r = {"build_s": round(time.time() - t0, 2),
             "build_ms": dict(zip(("graph", "prune", "merge"), (round(v, 1) for v in ix.meta()["build_ms"])))}
        if extra:
            ids, _, iters, upd, ms = kb.debug_cagra_knn_graph(xb_d, "L2", dict(extra, intermediate_graph_degree=igd))
            g0 = ids[torch.from_numpy(rows).to(dev)].cpu().numpy()
            hit = 0
            for i, a, b in zip(rows, g0, g0_gt):
                hit += len(np.intersect1d(a, b[b != i][:m]))
            r.update(iterations=iters, updates=upd.tolist(), graph_ms=round(ms, 1), g0_recall=round(hit / (len(rows) * m), 4))
            del ids
        for itopk in (32, 64, 128):
            for width in (1, 4):
                cfg = {"itopk_size": itopk, "search_width": width}
                ms, (ids, _) = timed(torch, lambda: ix.search(xq_d, k, cfg), args.reps)
                r[f"itopk{itopk}_w{width}"] = {"qps": round(args.nq / (ms * 1e-3)),
                                               "recall_at_10": round(recall(gt, ids.cpu().numpy()), 4)}
        res[name] = r
        print(json.dumps({name: r}), file=sys.stderr, flush=True)
        del ix
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

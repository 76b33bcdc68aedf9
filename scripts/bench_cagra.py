#!/usr/bin/env python3
"""GPU_CAGRA build and search (DESIGN §4.12, §6):

  1M x 128 datagen.clustered (L2), nq 10000, k 10, intermediate_graph_degree 128, graph_degree 64

Build time, split into the k-NN graph, the pruning and the merge (CUDA events, from the index meta).  For itopk_size in
{32, 64, 128, 256} x search_width in {1, 4}: device time of one batch (median of --reps after a warm-up, CUDA events),
queries/s, recall@10 against the exact FLAT search, and mean ndis per query.  Comparison points: the GPU HNSW on the same
data (M 32, efConstruction 100, GPU builder) over a sweep of ef, and baseline faiss IndexHNSWFlat::search (the oracle's
faiss::read_index of the GPU_CAGRA graph's IHNf stream; not the reference's own HNSW searcher) for the first
--ref-queries queries at efSearch 64 and 128, when the oracle is built.  The card
name and power limit are read in the same run.  Prints one JSON line.

  python scripts/bench_cagra.py [--rows 1000000] [--nq 10000] [--reps 5] [--ref-queries 1000]
"""
import argparse
import json
import os
import struct
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402

from bench_large_k import card  # noqa: E402


def recall(gt, ids):
    hit = sum(len(np.intersect1d(a, b[b >= 0], assume_unique=True)) for a, b in zip(gt, ids))
    return hit / float(gt.size)


def timed(torch, fn, reps):
    fn()                                               # warm-up: allocations, kernel attributes
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-queries", type=int, default=1000)
    args = ap.parse_args()
    import torch

    import knowhere_b200 as kb
    from knowhere_b200 import datagen
    n, d, k = args.rows, 128, 10
    dev = torch.device("cuda", 0)
    xb = datagen.clustered(n, d, 42)
    xq = datagen.clustered(args.nq, d, 43)
    gpu, power = card()
    res = {"gpu": gpu, "power_limit_w": power, "rows": n, "nq": args.nq, "k": k}
    xb_d = torch.from_numpy(xb).to(dev)
    xq_d = torch.from_numpy(xq).to(dev)
    flat = kb.Index("FLAT", "L2", d)
    flat.add(xb_d)
    gt = flat.search(xq_d, k)[0].cpu().numpy()
    del flat

    t0 = time.time()
    ix = kb.Index("GPU_CAGRA", "L2", d, {"intermediate_graph_degree": 128, "graph_degree": 64})
    ix.build(xb_d)
    res["cagra_build_s"] = round(time.time() - t0, 2)
    res["cagra_build_ms"] = dict(zip(("knn", "prune", "merge"), (round(v, 1) for v in ix.meta()["build_ms"])))
    for itopk in (32, 64, 128, 256):
        for width in (1, 4):
            cfg = {"itopk_size": itopk, "search_width": width}
            ms, (ids, _) = timed(torch, lambda: ix.search(xq_d, k, cfg), args.reps)
            ndis, nhops = ix.hnsw_last_stats()
            row = {"batch_ms": round(ms, 3), "qps": round(args.nq / (ms * 1e-3)), "recall_at_10": round(recall(gt, ids.cpu().numpy()), 4),
                   "ndis_per_query": round(ndis / args.nq, 1), "nhops_per_query": round(nhops / args.nq, 1)}
            res[f"cagra_itopk{itopk}_w{width}"] = row
            print(json.dumps({f"cagra_itopk{itopk}_w{width}": row}), file=sys.stderr, flush=True)

    if args.ref_queries > 0:
        from oracle import ref
        if ref.available():
            blob = ix.serialize_faiss()
            nr = min(args.ref_queries, args.nq)
            for ef in (64, 128):
                # efSearch in the HNSW header (after entry_point 0, max_level 0, efConstruction 128)
                old = struct.pack("<5i", 0, 0, 128, 16, 1)
                if blob.count(old) != 1:
                    raise SystemExit("efSearch field not found exactly once in the IHNf stream")
                b2 = blob.replace(old, struct.pack("<5i", 0, 0, 128, ef, 1))
                t1 = time.time()
                I0 = ref.read_and_search(b2, xq[:nr], k)[0]
                wall = time.time() - t1
                res[f"faiss_cpu_on_cagra_graph_ef{ef}"] = {"queries": nr, "wall_s": round(wall, 2), "qps": round(nr / wall, 1),
                                                         "recall_at_10": round(recall(gt[:nr], I0), 4)}
                print(json.dumps({f"faiss_cpu_on_cagra_graph_ef{ef}": res[f"faiss_cpu_on_cagra_graph_ef{ef}"]}), file=sys.stderr, flush=True)
        else:
            res["faiss_cpu_on_cagra_graph"] = "not measured (oracle not built)"
    del ix

    t0 = time.time()
    hn = kb.Index("HNSW", "L2", d, {"M": 32, "efConstruction": 100})
    hn.build(xb)
    res["hnsw_build_s"] = round(time.time() - t0, 2)
    for ef in (10, 16, 32, 64, 128, 256):
        ms, (ids, _) = timed(torch, lambda: hn.search(xq_d, k, {"ef": ef}), args.reps)
        ndis, nhops = hn.hnsw_last_stats()
        row = {"batch_ms": round(ms, 3), "qps": round(args.nq / (ms * 1e-3)), "recall_at_10": round(recall(gt, ids.cpu().numpy()), 4),
               "ndis_per_query": round(ndis / args.nq, 1)}
        res[f"hnsw_ef{ef}"] = row
        print(json.dumps({f"hnsw_ef{ef}": row}), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

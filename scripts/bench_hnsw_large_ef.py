#!/usr/bin/env python3
"""HNSW search at large ef and k (DESIGN §4.7 hnsw_wide_kernel, §6):

  1M x 128 datagen.clustered, M 16, efConstruction 100, graph built on the GPU, nq 1000
  (ef, k) in (4096, 4096) [four-queries-per-CTA kernel, the comparison point], (8192, 8192), (16384, 16384), (16384, 10)

For each setting: device time of one batch (median of --reps after a warm-up, CUDA events), queries/s, recall@k against
the exact large-k FLAT search on the GPU, ndis / nhops, and the reference's CPU searcher on the same graph (its faiss
stream with efSearch = ef) for the first --ref-queries queries, split over --ref-threads threads (default: the CPU count;
one faiss::read_index per thread, since the reference searches one query per call).  The card name and power limit are read in the same run.
Prints one JSON line.

  python scripts/bench_hnsw_large_ef.py [--rows 1000000] [--nq 1000] [--reps 5] [--ref-queries 100]
"""
import argparse
import json
import os
import struct
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench_large_k import card  # noqa: E402

SETTINGS = [(4096, 4096), (8192, 8192), (16384, 16384), (16384, 10)]


def recall(gt, ids):
    hit = sum(len(np.intersect1d(a, b[b >= 0], assume_unique=True)) for a, b in zip(gt, ids))
    return hit / float(gt.size)


def with_ef_search(blob, g, efc, ef):
    """the faiss stream with the HNSW header's efSearch (after entry_point, max_level, efConstruction) set to ef"""
    old = struct.pack("<5i", g["entry_point"], g["max_level"], efc, 16, 1)
    assert blob.count(old) == 1, "efSearch field not found in the faiss stream"
    return blob.replace(old, struct.pack("<5i", g["entry_point"], g["max_level"], efc, ef, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-queries", type=int, default=100)
    ap.add_argument("--ref-threads", type=int, default=os.cpu_count() or 1)
    args = ap.parse_args()
    import torch

    import knowhere_b200 as kb
    from knowhere_b200 import datagen
    n, d, efc = args.rows, 128, 100
    dev = torch.device("cuda", 0)
    xb = datagen.clustered(n, d, 42)
    xq = datagen.clustered(args.nq, d, 43)
    gpu, power = card()
    res = {"gpu": gpu, "power_limit_w": power, "rows": n, "nq": args.nq, "nproc": os.cpu_count()}

    t0 = time.time()
    ix = kb.Index("HNSW", "L2", d, {"M": 16, "efConstruction": efc})
    ix.build(xb)
    res["build_s"] = round(time.time() - t0, 1)
    xq_d = torch.from_numpy(xq).to(dev)
    flat = kb.Index("FLAT", "L2", d)
    flat.add(torch.from_numpy(xb).to(dev))
    kmax = max(k for _, k in SETTINGS)
    gt = np.empty((args.nq, kmax), np.int64)
    for s in range(0, args.nq, 100):
        gt[s:s + 100] = flat.search(xq_d[s:s + 100], kmax)[0].cpu().numpy()
    del flat

    g = ix.hnsw_export()
    blob = ix.serialize_faiss() if args.ref_queries > 0 else None
    from oracle import ref
    for ef, k in SETTINGS:
        ix.search(xq_d, k, {"ef": ef})                     # warm-up: allocations, kernel attributes
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            ids, _ = ix.search(xq_d, k, {"ef": ef})
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        ms = float(np.median(times))
        ids = ids.cpu().numpy()
        ndis, nhops = ix.hnsw_last_stats()
        row = {"engine": ix.last_stage_info()["engine"], "batch_ms": round(ms, 2), "qps": round(args.nq / (ms * 1e-3), 1),
               f"recall_at_{k}": round(recall(gt[:, :k], ids), 4), "ndis_per_query": ndis // args.nq,
               "nhops_per_query": nhops // args.nq}
        if args.ref_queries > 0:
            nr, nt = min(args.ref_queries, args.nq), args.ref_threads
            b2 = with_ef_search(blob, g, efc, ef)
            parts = np.array_split(np.arange(nr), nt)
            t1 = time.time()
            with ThreadPoolExecutor(nt) as ex:
                outs = list(ex.map(lambda p: ref.read_and_search(b2, xq[p], k)[0], [p for p in parts if len(p)]))
            wall = time.time() - t1
            I0 = np.concatenate(outs)
            row.update({"ref_queries": nr, "ref_threads": nt, "ref_wall_s": round(wall, 2),
                        "ref_qps": round(nr / wall, 1), f"ref_recall_at_{k}": round(recall(gt[:nr, :k], I0), 4),
                        "ref_same_ids": round(float((I0 == ids[:nr]).mean()), 4)})
        res[f"ef{ef}_k{k}"] = row
        print(json.dumps({f"ef{ef}_k{k}": row}), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

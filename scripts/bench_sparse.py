"""Sparse search throughput on the GPU (DESIGN §6): SPARSE_INVERTED_INDEX over two seeded workloads from datagen, nq 10000,
k 10 and 1000.  Prints one JSON line with the card name and power limit read in the same run.

  SPLADE-like: 1M rows, vocabulary 30522 with Zipf term frequencies, about 120 nonzeros per row, queries of about 40.
  BM25-like:   1M rows of integer term counts over 200k hashed uint32 terms, queries of 4-8 terms with IDF weights.

Device ms per batch are CUDA events around the search (median of the timed repeats after a warm-up); the postings and
bytes read come from last_search_counters.  The search reads every posting of every kept query term once per (query,
tile) it falls in, so it is bound by memory traffic: the share is the posting bytes over the time at 3.35 TB/s.  The CPU
comparison point is a numpy float64 brute force over a subset of the queries (one pass over the base's nonzeros each)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import knowhere_b200 as kb  # noqa: E402
from knowhere_b200 import datagen  # noqa: E402

PEAK_BW = 3.35e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:   # the numbers stay valid; the card is then unnamed in the output
        return f"unknown ({e})", "unknown"


def cpu_brute_force(base, queries, nq, k, metric, cfg):
    """numpy float64 brute force of the first nq queries: every row scored by one pass over the base's nonzeros"""
    ip, ix, val = base
    v64 = val.astype(np.float64)
    starts = ip[:-1]
    if metric == "BM25":
        k1, b, avg = cfg["bm25_k1"], cfg["bm25_b"], max(cfg["bm25_avgdl"], 1.0)
        L = np.add.reduceat(v64, starts) if v64.size else np.zeros(starts.size)
        L[np.diff(ip) == 0] = 0.0
    qp, qi, qv = queries
    ids = np.empty((nq, k), np.int64)
    for q in range(nq):
        t, w = qi[qp[q]:qp[q + 1]], qv[qp[q]:qp[q + 1]].astype(np.float64)
        pos = np.minimum(np.searchsorted(t, ix), t.size - 1)
        hit = t[pos] == ix
        c = np.where(hit, w[pos] * v64, 0.0)
        if metric == "BM25":
            rows = np.repeat(np.arange(starts.size), np.diff(ip))
            c = np.where(hit, w[pos] * (k1 + 1) * v64 / (v64 + k1 * (1 - b) + k1 * b / avg * L[rows]), 0.0)
        s = np.add.reduceat(c, starts)
        s[np.diff(ip) == 0] = 0.0
        top = np.lexsort((np.arange(s.size), -s))[:k]
        ids[q] = np.where(s[top] > 0, top, -1)
    return ids


def run(name, base, queries, metric, cfg, ks, reps, cpu_q):
    import torch
    ix = kb.Index("SPARSE_INVERTED_INDEX", metric, 0, cfg)
    dev = lambda c: tuple(torch.from_numpy(a.astype(np.int64) if a.dtype == np.uint32 else a).cuda() for a in c)  # noqa: E731
    t0 = time.time()
    ix.add_sparse(dev(base))
    build_s = time.time() - t0
    dq = dev(queries)
    nq = queries[0].size - 1
    out = {"workload": name, "rows": base[0].size - 1, "nnz": int(base[0][-1]), "nq": nq, "query_nnz": int(queries[0][-1]),
           "build_s": round(build_s, 3)}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for k in ks:
        ix.search_sparse(dq, k, cfg)   # warm-up
        times = []
        for _ in range(reps):
            e0.record()
            ix.search_sparse(dq, k, cfg)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        c = ix.last_counters()
        ms = float(np.median(times))
        out[f"k{k}"] = {"ms_per_batch": round(ms, 3), "ms_spread": [round(min(times), 3), round(max(times), 3)],
                        "qps": round(nq / ms * 1e3), "postings": c["pairs"], "posting_bytes": c["code_bytes"],
                        "posting_GBps": round(c["code_bytes"] / ms / 1e6, 1),
                        "share_of_3.35TBps": round(c["code_bytes"] / (ms * 1e-3) / PEAK_BW, 4)}
    ids, _ = ix.search_sparse(queries, 10, cfg)
    t0 = time.time()
    ref = cpu_brute_force(base, queries, cpu_q, 10, metric, cfg)
    out["cpu_numpy_f64_ms_per_query"] = round((time.time() - t0) / cpu_q * 1e3, 1)
    out["recall10_vs_f64"] = round(datagen.recall(ref, ids[:cpu_q]), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-queries", type=int, default=8)
    a = ap.parse_args()
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "workloads": []}
    base = datagen.sparse_splade(a.rows, 120, 1)
    queries = datagen.sparse_splade(a.nq, 40, 2)
    res["workloads"].append(run("splade", base, queries, "IP", {}, (10, 1000), a.reps, a.cpu_queries))
    del base, queries
    base, avgdl = datagen.sparse_bm25_docs(a.rows, 3)
    queries = datagen.sparse_bm25_queries(a.nq, a.rows, 4)
    cfg = {"bm25_k1": 1.2, "bm25_b": 0.75, "bm25_avgdl": avgdl}
    res["workloads"].append(run("bm25", base, queries, "BM25", cfg, (10, 1000), a.reps, a.cpu_queries))
    print(json.dumps(res))


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""IVF_PQ search across nprobe, past the 1008 probes of one coarse window (DESIGN §4.9.1):

  ivf_pq_1m   1M x 128, m 16, refine (fp32 store), refine_k 4 (bench.py's), nlist 8192
  ivf_pq_10m  10M x 128, the same, nlist 16384

nlist is raised above bench.py's so that 4096 probes are a fraction of the lists.  For nprobe 64, 512, 1008, 2048, 4096
and nlist, at nq queries and k 10: QPS from device events around the search (median of --reps), recall@10 against the
exact top-10 (FLAT), the engine that ran and the search counters.  The card name and power limit are read in the same
run.  Prints one JSON line.

  python scripts/bench_large_nprobe.py [--workloads ivf_pq_1m,ivf_pq_10m] [--nq 1000] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

WORKLOADS = {"ivf_pq_1m": (1_000_000, 8192), "ivf_pq_10m": (10_000_000, 16384)}
NPROBES = [64, 512, 1008, 2048, 4096]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0])
    except Exception:
        power = None
    return name, power


def timed(torch, fn, reps):
    fn()                                                  # warm-up: scratch allocations, kernel attributes
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="ivf_pq_1m,ivf_pq_10m")
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    import knowhere_b200 as kb
    from knowhere_b200 import datagen
    dev = torch.device("cuda", 0)
    gpu, power = card()
    res = {"gpu": gpu, "power_limit_w": power, "nq": args.nq, "k": 10}
    for name in args.workloads.split(","):
        n, nlist = WORKLOADS[name]
        d, k = 128, 10
        xb = datagen.clustered_torch(n, d, 42, dev)
        xq = datagen.clustered_torch(args.nq, d, 43, dev)
        gt, _ = kb.brute_force_search(xb, xq, k, "L2")
        gt = np.asarray(gt.cpu() if hasattr(gt, "cpu") else gt)
        ix = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": 16, "nbits": 8, "refine": True, "refine_type": "flat"})
        ix.build(xb)
        rows = []
        for nprobe in NPROBES + [nlist]:
            out = {}

            def run():
                out["r"] = ix.search(xq, k, {"nprobe": nprobe, "refine_k": 4})
            ms = timed(torch, run, args.reps)
            ids = out["r"][0]
            ids = np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids)
            rows.append({"nprobe": nprobe, "ms": round(ms, 3), "qps": round(args.nq / (ms * 1e-3)),
                         "recall_at_10": round(datagen.recall(gt, ids), 4), "engine": ix.last_stage_info()["engine"],
                         "counters": ix.last_counters()})
        res[name] = {"rows": n, "nlist": nlist, "sweep": rows}
        del ix, xb
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
